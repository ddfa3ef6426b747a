"""hrag_ppr_f64 (float64 PPR by iterative refinement with an fp64 residual sweep) against float64 oracles:
closed forms, MuSiQue-1k, operators fp32 cannot hold, PRPACK's Gauss-Seidel restatement on a graph with a
long-row hub, batching / determinism, the call contract, and accelerate(run_ppr_fp64=True)."""
import numpy as np
import pytest

from oracle import ppr, prpack_gs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def _engine(hb, n, src, dst, w):
    e = hb.Engine(0)
    e.load_graph(n, src, dst, w)          # the library's COO ingest keeps the fp64 (lo) plane
    return e


def _oracle_P(n, src, dst, w):
    return ppr.transition_matrix(ppr.symmetric_weights(n, src, dst, w))[0]


def _l1(a, b):
    return np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64)).sum(axis=-1)


def _order_ok(pi, o, tol):
    """Every pair whose oracle scores differ by more than 2 tol comes out in the oracle's order."""
    idx = np.argsort(-o, kind="stable")
    os_, ps = o[idx], pi[idx]
    suffix_max = np.maximum.accumulate(ps[::-1])[::-1]
    first_below = np.searchsorted(-os_, -(os_ - 2 * tol), side="right")    # first k with o_k < o_i - 2 tol
    has = first_below < len(os_)
    return bool(np.all(ps[has] > suffix_max[first_below[has]]))


def test_closed_forms(hb):
    e = _engine(hb, 2, [0], [1], [1.0])
    np.testing.assert_allclose(e.ppr_f64(np.array([1.0, 0.0])), [2 / 3, 1 / 3], rtol=0, atol=1e-13)
    # star: hub 1/(1-a^2), leaves a/3 of it
    e = _engine(hb, 4, [0, 0, 0], [1, 2, 3], [1, 1, 1])
    hub = 1 / 0.75
    leaf = 0.5 / 3 * hub
    tot = hub + 3 * leaf
    np.testing.assert_allclose(e.ppr_f64(np.array([1.0, 0, 0, 0])), [hub / tot] + [leaf / tot] * 3, rtol=0, atol=1e-13)
    # path 0-1-2 seeded at 0: (I - aP) x = e0 gives x = (7/6, 2/3, 1/6)
    e = _engine(hb, 3, [0, 1], [1, 2], [1.0, 1.0])
    np.testing.assert_allclose(e.ppr_f64(np.array([1.0, 0, 0])), [7 / 12, 1 / 3, 1 / 12], rtol=0, atol=1e-13)
    # an isolated seed keeps all its mass, an isolated non-seed gets none
    e = _engine(hb, 4, [0], [1], [1.0])
    np.testing.assert_allclose(e.ppr_f64(np.array([0.0, 0, 1, 0])), [0, 0, 1, 0], rtol=0, atol=1e-13)
    out = e.ppr_f64(np.array([[1.0, 0, 1, 0], [0, 0, 0, 2.0]]))
    # x = (4/3, 2/3, 1, 0) for the first reset: the isolated seed's mass is not amplified by 1 / (1 - a)
    np.testing.assert_allclose(out, [[4 / 9, 2 / 9, 1 / 3, 0], [0, 0, 0, 1]], rtol=0, atol=1e-13)


def _musique_resets(golden):
    n = int(golden["n_nodes"])
    R = np.zeros((64, n))
    R[:, golden["passage_vid"]] = golden["ref_passage_reset"].astype(np.float64)
    for q in range(64):
        for v, w in zip(golden["ref_seed_vid"][q], golden["ref_seed_w"][q]):
            if v >= 0:
                R[q, v] += w
    return R


def test_musique1k_against_sparse_lu(hb, golden):
    n = int(golden["n_nodes"])
    a = float(golden["damping"])
    e = _engine(hb, n, golden["edge_src"], golden["edge_dst"], golden["edge_w"])
    R = _musique_resets(golden)
    lu = ppr.factorize(golden["P"], a)
    O = np.stack([ppr.ppr_direct(golden["P"], r, a, lu=lu) for r in R])
    pv = golden["passage_vid"]

    def criterion(pi, tol):
        return [bool(_l1(pi[q], O[q]) <= tol and _order_ok(pi[q, pv], O[q, pv], tol)) for q in range(64)]

    for tol in (0.0, 1e-12):
        pi = e.ppr_f64(R, a, tol=tol)
        assert pi.dtype == np.float64 and pi.shape == R.shape
        want = tol or 1e-10
        assert np.all(criterion(pi, want)), (tol, _l1(pi, O).max())
        st = e.stats()
        assert st["ppr_error_bound"] <= want
        assert st["ppr_error_bound"] >= _l1(pi, O).max()
    # the fp32 solver cannot meet the same criterion on this graph
    pi32 = e.ppr(R.astype(np.float32), a)
    assert not all(criterion(pi32.astype(np.float64), 1e-10))


def test_operator_not_representable_in_fp32(hb):
    from hipporag_b200.engine import build_transition_csr
    rng = np.random.default_rng(11)
    # vertices 0, 1, 2 have strengths 3, 7 and 11 (unit edges); the rest carry synonymy-style weights over three decades
    src = [0] * 3 + [1] * 7 + [2] * 11
    dst = list(range(3, 6)) + list(range(6, 13)) + list(range(13, 24))
    m = 600
    src += rng.integers(3, 200, m).tolist()
    dst += rng.integers(3, 200, m).tolist()
    w = np.concatenate([np.ones(21), 10.0 ** rng.uniform(-3, 0, m)])
    n = 200
    P = _oracle_P(n, src, dst, w)
    assert np.any(P.data != P.data.astype(np.float32))
    R = np.zeros((5, n))
    R[0, 0] = R[1, 1] = R[2, 2] = 1.0
    R[3, 3:40] = rng.random(37)
    R[4] = rng.random(n)
    O = np.stack([ppr.ppr_direct(P, r, 0.5) for r in R])
    for eng in (_engine(hb, n, src, dst, w), hb.Engine(0)):
        if eng.n_nodes == 0:          # the same operator through load_graph_csr with float64 values
            eng.load_graph_csr(n, *build_transition_csr(n, src, dst, w, dtype=np.float64))
        pi = eng.ppr_f64(R, 0.5, tol=1e-12)
        assert _l1(pi, O).max() <= 1e-12, _l1(pi, O)
    # a graph loaded from fp32 values has no fp64 operator: the solve refuses instead of assuming lo = 0
    e32 = hb.Engine(0)
    e32.load_graph_csr(n, *build_transition_csr(n, src, dst, w))
    with pytest.raises(hb.HragError, match="hrag_load_graph_csr_f64 or hrag_load_graph_coo"):
        e32.ppr_f64(R[0])


def _powerlaw_graph(seed=5):
    """A hub with 400 distinct neighbours (a long row: segment path), a heavy-tailed rest, self-loops, parallel
    edges and isolated vertices (sinks)."""
    rng = np.random.default_rng(seed)
    n = 1500
    core = n - 40                                         # the last 40 vertices stay isolated
    hub_nb = rng.choice(np.arange(1, core), 400, replace=False)
    p = 1.0 / np.arange(1, core + 1) ** 0.9
    p /= p.sum()
    a, b = rng.choice(core, 4000, p=p), rng.integers(0, core, 4000)
    loops = rng.integers(0, core, 30)
    src = np.concatenate([np.zeros(400, np.int64), a, loops, a[:300]])
    dst = np.concatenate([hub_nb, b, loops, b[:300]])     # a[:300] / b[:300] again: parallel edges
    w = np.concatenate([rng.uniform(0.5, 2.0, 400), 10.0 ** rng.uniform(-2, 0.5, 4000), rng.uniform(0.1, 1, 30),
                        rng.uniform(0.1, 1, 300)])
    return n, src, dst, w


@pytest.mark.parametrize("damping", [0.5, 0.85])
def test_against_prpack_gauss_seidel(hb, damping):
    n, src, dst, w = _powerlaw_graph()
    e = _engine(hb, n, src, dst, w)
    rng = np.random.default_rng(1)
    R = np.zeros((3, n))
    R[0, 0] = 1.0                                         # the hub itself
    R[1, rng.integers(0, n - 40, 12)] = rng.random(12)
    R[1, n - 1] = 0.3                                     # a seed on a sink
    R[2] = rng.random(n)
    pi = e.ppr_f64(R, damping)
    for q in range(3):
        want = prpack_gs.personalized_pagerank_gs(n, src, dst, w, R[q], damping)
        assert _l1(pi[q], want) <= 2e-10, (q, _l1(pi[q], want))
    P = _oracle_P(n, src, dst, w)
    O = np.stack([ppr.ppr_direct(P, r, damping) for r in R])
    assert _l1(pi, O).max() <= e.stats()["ppr_error_bound"] <= 1e-10


@pytest.fixture(scope="module")
def kg8k(hb):
    from hipporag_b200 import synth
    kg = synth.make_kg(8000, 80000, seed=2)
    lu = ppr.factorize(_oracle_P(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w), 0.5)
    return kg, _engine(hb, kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w), lu


@pytest.mark.parametrize("B", [1, 7, 16, 17, 40])
def test_batching_and_determinism(hb, kg8k, B):
    kg, e, lu = kg8k
    n = kg.n_nodes
    rng = np.random.default_rng(B)
    R = np.zeros((B, n))
    for q in range(B):
        R[q, rng.integers(0, n, 6)] = rng.random(6)
    R[B // 2, kg.passage_vid] = 0.05 * rng.random(kg.n_pass)     # one query with a dense reset (needs more work)
    out = e.ppr_f64(R)
    again = e.ppr_f64(R)
    assert out.tobytes() == again.tobytes()
    perm = rng.permutation(B)[::-1].copy()
    shuffled = e.ppr_f64(R[perm])
    assert shuffled.tobytes() == out[perm].tobytes()
    P = _oracle_P(n, kg.edge_src, kg.edge_dst, kg.edge_w)
    for q in {0, B // 2, B - 1}:
        assert _l1(out[q], ppr.ppr_direct(P, R[q], 0.5, lu=lu)) <= 1e-10
    # the same query at other batch widths agrees within the bound (the width changes only summation order)
    single = e.ppr_f64(R[B // 2])
    assert _l1(single, out[B // 2]) <= 2e-10


def test_contract(hb):
    from hipporag_b200 import synth
    kg = synth.make_kg(3000, 30000, seed=9)
    n = kg.n_nodes
    e = _engine(hb, n, kg.edge_src, kg.edge_dst, kg.edge_w)
    P = _oracle_P(n, kg.edge_src, kg.edge_dst, kg.edge_w)
    rng = np.random.default_rng(3)
    r = np.zeros(n)
    r[rng.integers(0, n, 20)] = rng.random(20)
    dirty = r.copy()
    zeros = np.flatnonzero(r == 0)
    dirty[zeros[:10]] = np.nan
    dirty[zeros[10:20]] = -3.0
    clean = e.ppr_f64(r)
    np.testing.assert_array_equal(e.ppr_f64(dirty), clean)          # NaN and negative entries count as 0
    assert abs(clean.sum() - 1.0) <= 1e-13
    for a, tol in ((0.5, 0.0), (0.5, 1e-12), (0.85, 1e-11)):
        pi = e.ppr_f64(r, a, tol=tol)
        st = e.stats()
        err = _l1(pi, ppr.ppr_direct(P, r, a))
        assert err <= st["ppr_error_bound"] <= (tol or 1e-10), (a, tol, err, st["ppr_error_bound"])
        # the bound is 2 ||r||_1 / ((1 - a) ||v||_1) of the reported relative residual
        assert st["ppr_error_bound"] == pytest.approx(2.0 * st["ppr_residual"] / (1.0 - a), rel=1e-12, abs=0)
    with pytest.raises(hb.HragError, match="1e-13"):
        e.ppr_f64(r, tol=5e-14)
    with pytest.raises(hb.HragError, match="1e-13"):
        e.ppr_f64(r, tol=-1.0)


def test_sharded_handle_rejects(hb):
    """world > 1 is refused; a single-process NCCL communicator of world 2 is enough to get there (no peer joins,
    so nothing collective may run: the check must come first)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("a world > 1 handle needs two GPUs")
    import multiprocessing as mp
    ctx = mp.get_context("spawn")
    with ctx.Pool(2) as pool:
        uid = hb.Engine.new_comm_id()
        msgs = pool.starmap(_rank_rejects, [(uid, 0), (uid, 1)])
    for m in msgs:
        assert "world > 1" in m, m


def _rank_rejects(uid, rank):
    import hipporag_b200 as hb
    e = hb.Engine(rank, shard_mode=1)
    e.init_comm(uid, rank, 2)
    e.load_graph(4, [0, 1], [1, 2], [1.0, 1.0])
    try:
        e.ppr_f64(np.array([1.0, 0, 0, 0]))
    except hb.HragError as ex:
        return str(ex)
    return "no error"


def test_accelerate_run_ppr_fp64(hb):
    import tempfile
    from tests import fake_hipporag
    from hipporag_b200 import synth
    fake_hipporag.install_stub_package()
    kg = synth.make_kg(3000, 30000, seed=5)
    fe, pe = synth.unit_rows(kg.n_facts, 64, 1), synth.unit_rows(kg.n_pass, 64, 2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 2, seed=3)
    P = _oracle_P(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    r = np.zeros(kg.n_nodes)
    r[kg.passage_vid[:5]] = 1.0
    r[7] = 2.0
    want = ppr.ppr_direct(P, r, 0.5)[kg.passage_vid]
    with tempfile.TemporaryDirectory() as wd:
        got = []
        for _ in range(2):                                  # cache miss, then cache hit
            rag = fake_hipporag.FakeRag(kg, fe, pe, qf, qp, ["a", "b"])
            rag.working_dir = wd
            hb.accelerate(rag, device=0, run_ppr_fp64=True)
            order, scores = rag.run_ppr(r, 0.5)
            assert scores.dtype == np.float64
            assert np.array_equal(order, np.lexsort((np.arange(want.shape[0]), -want)))
            np.testing.assert_allclose(scores, want[order], rtol=1e-12, atol=0)
            got.append((order.tobytes(), scores.tobytes(), rag._b200_state["cache_hit"]))
        assert got[0][2] is False and got[1][2] is True
        assert got[0][:2] == got[1][:2]
        # default mode is the fp32 run_ppr
        rag = fake_hipporag.FakeRag(kg, fe, pe, qf, qp, ["a", "b"])
        hb.accelerate(rag, device=0)
        ids32, sc32 = rag.run_ppr(r, 0.5)
        eng = hb.Engine(0)
        eng.load_graph_csr(kg.n_nodes, *hb.build_transition_csr(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w))
        pi32 = eng.ppr(r.astype(np.float32), 0.5)[kg.passage_vid].astype(np.float64)
        assert np.array_equal(ids32, np.lexsort((np.arange(pi32.shape[0]), -pi32)))
        np.testing.assert_array_equal(sc32, pi32[ids32])
