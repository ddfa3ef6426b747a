// The PPR solvers: sweep planning, the fp32 solver, the mixed-precision solver (fp16 state, one refinement round, a
// CUDA-graph cache of its solves) and float64 refinement; hrag_ppr, hrag_ppr_f64 and hrag_plan_sweeps.
#include <algorithm>
#include <cmath>
#include <cstring>

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

int ensure_state_mixed(hrag_t* h) {
    const size_t rows = state_rows(h);
    const size_t hb = rows * 32 * 2;
    if (h->slab.p == nullptr || h->slab_hb != hb) {
        HRAG_CHECK(!h->p2p, "internal: the state slab cannot change after hrag_p2p_import");
        h->slab.reset();
        HRAG_TRY(h->slab.ensure(5 * hb + 256));
        HRAG_CUDA(cudaMemset(static_cast<char*>(h->slab.p) + 5 * hb, 0, 256));      // epoch flags
        h->slab_hb = hb;
        for (int i = 0; i < 4; ++i) h->H[i] = static_cast<char*>(h->slab.p) + (size_t)i * hb;
        h->H0b = static_cast<char*>(h->slab.p) + 4 * hb;
        if (!h->p2p_err.p) HRAG_TRY(h->p2p_err.zeros(sizeof(int)));
        if (!h->done_ctr.p) HRAG_TRY(h->done_ctr.zeros(sizeof(unsigned int)));
    }
    HRAG_TRY(h->partials.ensure((size_t)std::max(mixed_partial_rows(h->g), 1024) * 32 * sizeof(float)));
    HRAG_TRY(h->sums.ensure(320 * sizeof(double)));      // sums of x0, of d, of |r| (x2), and of v (four sets)
    HRAG_TRY(h->mixed_aux.ensure(32 * sizeof(float)));   // column scales, set 0
    // [0] running max of the measured residual (float), [1] fp16 overflow flag (int)
    if (h->rho.p == nullptr) HRAG_TRY(h->rho.zeros(2 * sizeof(float)));
    return 0;
}

int ensure_state_pair(hrag_t* h) {
    HRAG_CHECK(h->world == 1, "internal: paired solves run on a single GPU");
    const size_t hb2 = (size_t)h->g.n_global * 64 * 2;
    HRAG_TRY(h->slab_pair.ensure(5 * hb2));
    for (int i = 0; i < 4; ++i) h->HP[i] = static_cast<char*>(h->slab_pair.p) + (size_t)i * hb2;
    h->HP0b = static_cast<char*>(h->slab_pair.p) + 4 * hb2;
    HRAG_TRY(h->partials_b.ensure(h->partials.cap));
    return 0;
}

// Compact right-hand-side buffers of stage B (two sets, four for paired solves; see the handle) + the node -> slot
// tables.
int ensure_compact_rhs(hrag_t* h, int n_sets) {
    const size_t n_slots = (size_t)h->t.n_passages + 32 * kSeedSlots;
    for (int s = 0; s < n_sets; ++s) {
        HRAG_TRY(h->slot_map[s].ensure((size_t)h->g.n_global * sizeof(int)));
        HRAG_TRY(h->slot_vid[s].ensure(n_slots * sizeof(int)));
        HRAG_TRY(h->Vc[s].ensure(n_slots * 32 * sizeof(float)));
        HRAG_TRY(h->R16[s].ensure(n_slots * 32 * 2));
    }
    HRAG_TRY(h->mixed_aux1.ensure(3 * 32 * sizeof(float)));
    HRAG_TRY(h->prep_scratch.ensure((size_t)std::max(compact_rhs_partial_rows(h->t.n_passages), 1024) * 32 * sizeof(float)));
    if (!h->slot_maps_valid) {                       // a graph or table load invalidated every set
        h->slot_maps_built = 0;
        h->slot_maps_valid = true;
    }
    for (; h->slot_maps_built < n_sets; ++h->slot_maps_built)
        HRAG_TRY(slot_map_build(h->g.n_global, h->t.n_passages, h->t.passage_vid,
                                h->slot_map[h->slot_maps_built].as<int>(), h->stream));
    return 0;
}

float* set_scale(hrag_t* h, int set) {
    return set == 0 ? h->mixed_aux.as<float>() : h->mixed_aux1.as<float>() + 32 * (set - 1);
}

int resolve_spans(hrag_t* h) {
    HRAG_CUDA(cudaStreamSynchronize(h->stream));
    if (h->p2p && h->p2p_err.p) {
        int err = 0;
        HRAG_CUDA(cudaMemcpy(&err, h->p2p_err.p, sizeof(int), cudaMemcpyDeviceToHost));
        if (err != 0) HRAG_CUDA(cudaMemset(h->p2p_err.p, 0, sizeof(int)));   // report once; this call's results are invalid
        HRAG_CHECK(err == 0, "node-range sharding: a peer GPU never published its rows (fused exchange timed out); "
                             "the results of this call are invalid");
    }
    if ((h->rho_dirty || h->check_tol > 0.0) && h->rho.p) {
        // every mixed solve of this call (a fresh capture or a replayed graph) raised rho[0] = the running maximum of
        // the measured relative L1 residual of its fp16 first solve, and rho[1] if an fp16 iterate left fp16's range.
        // Both are cleared here, checked call or not, so the next call is judged by its own solves only.
        float rho[2] = {0.f, 0.f};
        HRAG_CUDA(cudaMemcpy(rho, h->rho.p, sizeof(rho), cudaMemcpyDeviceToHost));
        HRAG_CUDA(cudaMemset(h->rho.p, 0, sizeof(rho)));
        int overflow = 0;
        memcpy(&overflow, &rho[1], sizeof(int));
        const double tol = h->check_tol, kappa = h->check_kappa;
        h->check_tol = h->check_kappa = 0.0;
        h->rho_dirty = false;
        if (overflow) {
            set_error("PPR (mixed solver): an fp16 iterate reached 65520 in magnitude and would have been clamped, so "
                      "the result is invalid -- pass more sweeps (iters) or use HRAG_PPR_FP32");
            return 5;
        }
        if (tol > 0.0) {
            // a-posteriori check of the mixed solver: the refinement round contracts rho by kappa (plan_sweeps)
            h->last_rho = rho[0];
            h->last_bound = (float)(rho[0] * kappa);
            if (!(rho[0] * kappa <= 10.0 * tol)) {
                set_error("PPR (mixed solver): measured relative residual " + std::to_string(rho[0]) +
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

// Sub-batch k's part of a [N, 2, 32] pair buffer (64 B into each row for k = 1); null stays null.
static void* pair_half(const void* p, int k) {
    return p ? static_cast<char*>(const_cast<void*>(p)) + 64 * k : nullptr;
}

// One sweep of the n sub-batches of a solve (n = 2: one paired walk over the interleaved buffers x, prev, y).
// slot_map / rhs / v32 / scale are per sub-batch; a dense rhs (slot_map null) is a buffer like x.  final: the column-sum
// partials of sub-batch k go to h->partials (k = 0) / h->partials_b (k = 1).
static int mixed_sweep_n(hrag_t* h, int n, int mode, const void* x, const int* const* slot_map,
                         const void* const* rhs, const float* const* v32, const float* const* scale, const void* prev,
                         void* y, float alpha, float w, float t, bool final, int* n_part) {
    if (n == 1)
        return mixed_sweep_x(h, mode, x, slot_map[0], rhs[0], v32[0], scale[0], prev, y, alpha, w, t,
                             final ? h->partials.as<float>() : nullptr, n_part);
    MixedSweepIO io[2];
    for (int k = 0; k < 2; ++k) {
        io[k].xh = pair_half(x, k);
        io[k].slot_map = slot_map[k];
        io[k].rhs_h = slot_map[k] ? rhs[k] : pair_half(rhs[k], k);
        io[k].v32 = v32[k];
        io[k].col_scale = scale[k];
        io[k].prevh = pair_half(prev, k);
        io[k].yh = pair_half(y, k);
        io[k].partials = final ? (k ? h->partials_b : h->partials).as<float>() : nullptr;
    }
    int* overflow = h->rho.p ? h->rho.as<int>() + 1 : nullptr;
    return mixed_sweep2(h->g, mode, io, alpha, w, t, n_part, overflow, h->stream);
}

// Column sums of sub-batch k of the last final sweep -> h->sums + off (+ kSumPair for k = 1)
static int mixed_sums(hrag_t* h, int n, int n_part, int off) {
    for (int k = 0; k < n; ++k)
        HRAG_TRY(colsum_reduce((k ? h->partials_b : h->partials).as<float>(), n_part, 32,
                               h->sums.as<double>() + off + (k ? kSumPair : 0), h->stream));
    return 0;
}

// m Chebyshev sweeps of the fp16 solver on (I - aP) x = rhs for n sub-batches, first iterate x_first (= rhs as a dense
// [N, 32] array, [N, 2, 32] for a pair); rhs[k] is addressed through slot_map[k] (null = dense).  Iterates alternate
// between bufA and bufC; *result = the last one, its column sums land in h->sums + sums_off.
static int mixed_cheb(hrag_t* h, int n, const int* const* slot_map, const void* const* rhs, void* x_first, void* bufA,
                      void* bufC, int m, float alpha, void** result, int sums_off) {
    HRAG_CHECK(m >= 1, "mixed solver: sweep count must be >= 1");
    const float* none[2] = {nullptr, nullptr};
    double w = 1.0;
    void *x = x_first, *prev = nullptr, *y = nullptr;
    int n_part = 0;
    for (int it = 1; it <= m; ++it) {
        const float wf = cheb_step(it, alpha, &w, bufA, bufC, prev, &y);
        HRAG_TRY(mixed_sweep_n(h, n, 0, x, slot_map, rhs, none, none, prev, y, alpha, wf, 1.f, it == m, &n_part));
        prev = x;
        x = y;
        h->stats.ppr_sweeps += n;
        h->stats.ppr_columns += 32 * n;
    }
    HRAG_TRY(mixed_sums(h, n, n_part, sums_off));   // local rows only: see dev_ppr_mixed_body
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
    double* sums = h->sums.as<double>();
    void* const* H = n == 2 ? h->HP : h->H;
    const int* slot_map[2] = {in[0].slot_map, n == 2 ? in[1].slot_map : nullptr};
    const void* rhs16[2] = {in[0].rhs16, n == 2 ? in[1].rhs16 : nullptr};
    const float* vexact[2] = {in[0].Vexact, n == 2 ? in[1].Vexact : nullptr};
    const float* scale[2] = {in[0].scale, n == 2 ? in[1].scale : nullptr};
    void* x0_dense = in[0].x0_dense;
    void* x0 = nullptr;
    void* d = nullptr;
    HRAG_TRY(mixed_cheb(h, n, slot_map, rhs16, x0_dense, H[1], H[2], plan.m1, alpha, &x0, kSumX0));
    void* other = (x0 == H[1]) ? H[2] : H[1];
    int n_part = 0;
    const void* none[2] = {nullptr, nullptr};
    HRAG_TRY(mixed_sweep_n(h, n, 1, x0, slot_map, none, vexact, scale, nullptr, H[3], alpha, 1.f, kMixedT, true,
                           &n_part));
    h->stats.ppr_sweeps += n;
    h->stats.ppr_columns += 32 * n;
    HRAG_TRY(mixed_sums(h, n, n_part, kSumR));
    const int* dense[2] = {nullptr, nullptr};
    const void* resid[2] = {H[3], H[3]};
    HRAG_TRY(mixed_cheb(h, n, dense, resid, H[3], x0_dense, other, plan.m2, alpha, &d, kSumD));
    if (h->world > 1) {      // node-range sharding: every rank summed its own rows -- ONE all-reduce for the three sums
        StageTimer tc(h, ST_COMM);
        HRAG_NCCL(g_nccl.AllReduce(sums, sums, 96, ncclDouble, ncclSum, h->comm, h->stream));
    }
    for (int k = 0; k < n; ++k) {
        const int off = k ? kSumPair : 0;
        HRAG_TRY(residual_check(sums + off + kSumR, in[k].vsum, in[k].scale, 1.f / kMixedT, h->rho.as<float>(),
                                h->stream));
        X0[k] = pair_half(x0, k);
        D[k] = pair_half(d, k);
    }
    return 0;
}

// The solve of one sub-batch is ~20 launches whose arguments depend only on the buffer set and the sweep plan, so on a
// single GPU it is captured once per (set, plan) into a CUDA graph and replayed (one launch per sub-batch instead of ~20:
// what bounds small real graphs like MuSiQue-1k, where a sweep is a few microseconds of work).  Multi-GPU runs (epoch
// values change per sweep) take the plain path.
int dev_ppr_mixed(hrag_t* h, const SweepPlan& plan, float alpha, int n, const MixedRhs* in, void** X0, void** D) {
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
        if (h->solve_graphs.size() >= 8) {                       // bounded cache: drop everything stale
            HRAG_CUDA(cudaStreamSynchronize(h->stream));         // none of them may still be executing
            for (auto& c : h->solve_graphs) cudaGraphExecDestroy(c.exec);
            h->solve_graphs.clear();
        }
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
            double* vsum = h->sums.as<double>() + kSumV;
            HRAG_TRY(mixed_prepare_rhs(h->V.as<float>(), (int64_t)N, damping, h->partials.as<float>(), vsum,
                                       h->mixed_aux.as<float>(), h->H[0], h->stream));
            MixedRhs in;
            in.Vexact = h->V.as<float>();
            in.rhs16 = in.x0_dense = h->H[0];
            in.scale = h->mixed_aux.as<float>();
            in.vsum = vsum;
            HRAG_TRY(dev_ppr_mixed(h, plan, damping, 1, &in, &X0, &D));
            HRAG_TRY(state_to_scores_mixed(X0, D, 1.f / kMixedT, nb, N, h->sums.as<double>(),
                                           h->sums.as<double>() + 32, h->d_scores.as<float>(), h->stream));
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
