"""A numpy model of the mixed-precision PPR solver of csrc/ppr_mixed.cu / solve.cu (fp16 STORAGE of every iterate and of
the scaled right-hand side, fp32 arithmetic, Chebyshev semi-iteration, one refinement round through the fp32 residual),
run with the sweep counts `hrag_plan_sweeps` derives, against the float64 oracle.  CPU only: it pins the NUMERICS of the
design -- the fp16 noise constant behind the a-priori plan, the residual the a-posteriori check reads, the accuracy after
one refinement round -- for dampings the GPU parity tests do not all visit.  (GPU: tests/test_gpu_parity.py.)"""
import numpy as np
import pytest

from oracle import ppr


def _h(x):
    return x.astype(np.float16).astype(np.float32)


def _cheb(P32, rhs, x0, m, a):
    """mixed_cheb: x1 = aPx0 + rhs; x_{k+1} = w (aPx_k + rhs) + (1 - w) x_{k-1}; every stored iterate rounded to fp16."""
    rho2, w = a * a, 1.0
    x, prev = x0, None
    for it in range(1, m + 1):
        y = np.float32(a) * (P32 @ x) + rhs
        if it >= 2:
            w = 1.0 / (1.0 - rho2 / 2.0) if it == 2 else 1.0 / (1.0 - rho2 * w / 4.0)
            y = np.float32(w) * y + np.float32(1.0 - w) * (x0 if it == 2 else prev)
        y = _h(y)
        prev, x = x, y
    return x


@pytest.mark.parametrize("damping", [0.3, 0.5, 0.7])
def test_fp16_state_plus_one_refinement_round_reaches_fp32_accuracy(damping):
    from hipporag_b200 import synth
    from hipporag_b200.engine import plan_sweeps
    kg = synth.make_kg(6000, 60000, seed=4)
    n = kg.n_nodes
    P = ppr.transition_matrix(ppr.symmetric_weights(n, kg.edge_src, kg.edge_dst, kg.edge_w))[0]
    P32 = P.astype(np.float32)
    rng = np.random.default_rng(0)
    B = 6
    R = np.zeros((n, B), np.float32)                             # HippoRAG's reset vectors: dense on passages + 5 phrases
    R[kg.passage_vid] = 0.05 * rng.random((kg.n_pass, B), dtype=np.float32)
    for b in range(B):
        R[rng.integers(0, kg.n_ent, 5), b] = rng.random(5, dtype=np.float32)
    R[:, 1] *= 1e-3                                              # a column on a very different scale
    plan = plan_sweeps(damping)
    assert plan["solver"] == "mixed"
    m1, _, m2 = plan["mixed_sweeps"]
    a = damping
    vs = R.sum(axis=0, dtype=np.float64)
    scale = np.exp2(np.floor(np.log2(32768.0 * (1.0 - a) / vs))).astype(np.float32)     # column_scale()
    rhs16 = _h(R * scale)
    x0 = _cheb(P32, rhs16, rhs16, m1, a)
    assert np.isfinite(x0).all() and x0.max() < 65504.0         # the scale makes fp16 overflow impossible
    t = np.float32(64.0)                                         # kMixedT
    r = _h(t * (np.float32(a) * (P32 @ x0) + (scale * R - x0)))  # MODE 1: fp32 residual of the fp16 iterate
    rho = float((np.abs(r).sum(axis=0, dtype=np.float64) / t / (scale * vs)).max())     # k_residual_check
    d = _cheb(P32, r, r, m2, a)
    x = x0.astype(np.float64) + d.astype(np.float64) / 64.0
    pi = x / x.sum(axis=0, keepdims=True)
    want = ppr.ppr_batch_power(P, R.astype(np.float64), a)
    # the fp16 noise model of plan_sweeps: a converged fp16 solve leaves ~2.5e-4 / (1 - a) of relative L1 residual
    noise = 2.5e-4 / (1.0 - a)
    assert 0.3 * noise < rho < 2.0 * noise
    # after one refinement round: fp32-level accuracy, well inside the predicted bound and the parity tolerances
    rel_l1 = np.abs(pi - want).sum(axis=0).max()
    assert rel_l1 < plan["predicted_error"] < 1e-6
    assert np.max(np.abs(pi - want) / want.max(axis=0, keepdims=True)) < 1e-6
    big = want > 1e-3 * want.max(axis=0, keepdims=True)
    assert np.max(np.abs(pi - want)[big] / want[big]) < 5e-6    # tests/util.py RTOL is 2e-5
    # without the refinement round the fp16 iterate alone is three orders of magnitude worse
    pi0 = x0.astype(np.float64) / x0.astype(np.float64).sum(axis=0, keepdims=True)
    assert np.abs(pi0 - want).sum(axis=0).max() > 100 * rel_l1
