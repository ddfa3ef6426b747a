"""BASELINE.json's full single-GPU size (C3: 1M nodes / 10M edges, 2.75M facts, 100k passages):
size-independent properties of the CUDA path plus a float64-oracle spot check.  Embedding width is
64 here (the 768-wide case is what bench.py times); everything else is the C3 shape."""
import numpy as np
import pytest

from oracle import ppr, retrieve
from tests.util import assert_topk_matches

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def c3():
    import hipporag_b200 as hb
    from hipporag_b200 import synth
    kg = synth.make_kg(1_000_000, 10_000_000, seed=0)
    d = 64
    fe = synth.unit_rows(kg.n_facts, d, seed=100)
    pe = synth.unit_rows(kg.n_pass, d, seed=101)
    qf, qp, planted = synth.make_queries(kg, fe, pe, 200, seed=7)
    r = hb.B200Retriever(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w, kg.passage_vid, kg.fact_subj_vid,
                         kg.fact_obj_vid, kg.ent_chunk_count, fe, pe)
    return hb, kg, fe, pe, qf, qp, planted, r


def test_full_size_output_invariants(c3):
    hb, kg, fe, pe, qf, qp, planted, r = c3
    ids, scores, fidx, fscore = r.retrieve(qf, qp, topk=200)
    assert ids.shape == (200, 200) and ids.min() >= 0 and ids.max() < kg.n_pass
    assert all(len(set(row.tolist())) == 200 for row in ids)                   # no duplicates
    assert np.all(np.diff(scores, axis=1) <= 0)                                # sorted, best first
    assert np.all(scores > 0) and np.all(scores.sum(axis=1) < 1.0)             # probabilities
    assert np.array_equal(fidx[:, 0], planted)                                 # the planted fact wins
    assert np.allclose(fscore[:, 0], 1.0)                                      # min-max: best fact = 1
    ids2, scores2, _, _ = r.retrieve(qf, qp, topk=200)                         # deterministic / idempotent
    assert np.array_equal(ids, ids2) and np.array_equal(scores, scores2)
    ids50, scores50, _, _ = r.retrieve(qf[:40], qp[:40], topk=50)              # top-50 = prefix of top-200
    assert np.array_equal(ids50, ids[:40, :50])
    np.testing.assert_allclose(scores50, scores[:40, :50], rtol=1e-6)


def test_full_size_ppr_is_a_normalised_linear_operator(c3):
    hb, kg, fe, pe, qf, qp, planted, r = c3
    rng = np.random.default_rng(0)
    n = kg.n_nodes
    R = np.zeros((34, n), np.float32)                                          # 34 > 16 -> mixed-precision solver
    for b in range(34):
        R[b, rng.integers(0, n, 50)] = rng.random(50, dtype=np.float32) + 0.1
    R[2] = R[0] + R[1]
    R[3] = 5.0 * R[0]
    pi = r.engine.ppr(R)
    np.testing.assert_allclose(pi.sum(axis=1), 1.0, atol=2e-5)
    assert pi.min() >= 0
    s0, s1 = R[0].sum(dtype=np.float64), R[1].sum(dtype=np.float64)
    mix = (s0 * pi[0].astype(np.float64) + s1 * pi[1].astype(np.float64)) / (s0 + s1)
    assert np.max(np.abs(pi[2] - mix)) / mix.max() < 2e-5                      # linearity in the reset vector
    assert np.max(np.abs(pi[3] - pi[0])) / pi[0].max() < 2e-5                  # scale invariance


def test_full_size_spot_check_against_the_oracle(c3):
    hb, kg, fe, pe, qf, qp, planted, r = c3
    ids, scores, _, _ = r.retrieve(qf[:40], qp[:40], topk=200)                 # batch > 16: default (mixed) solver
    P = ppr.transition_matrix(ppr.symmetric_weights(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w))[0]
    tb = retrieve.Tables(kg.n_nodes, kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    for q in (0, 17, 39):
        o = retrieve.retrieve_one(P, tb, fe, pe, qf[q], qp[q], top_k=None)
        full = np.empty(len(o["ids"]))
        full[o["ids"]] = o["scores"]
        assert_topk_matches(ids[q], scores[q], full, 200, what=f"C3 query {q}")


def test_full_size_768_wide_against_the_oracle():
    """The exact configuration bench.py times (C3 at d = 768): 40 queries through the default path (wgmma split
    GEMM with the fused selection epilogue, mixed-precision PPR), 8 of them checked against the float64 oracle --
    top-5 facts identical, top-200 passages and scores per tests/util.py."""
    import hipporag_b200 as hb
    from hipporag_b200 import synth
    kg = synth.make_kg(1_000_000, 10_000_000, seed=0)
    d = 768
    fe = synth.unit_rows(kg.n_facts, d, seed=100)
    pe = synth.unit_rows(kg.n_pass, d, seed=101)
    qf, qp, planted = synth.make_queries(kg, fe, pe, 40, seed=11)
    r = hb.B200Retriever(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w, kg.passage_vid, kg.fact_subj_vid,
                         kg.fact_obj_vid, kg.ent_chunk_count, fe, pe)
    ids, scores, fidx, fscore = r.retrieve(qf, qp, topk=200)
    st = r.engine.stats()
    assert st["ppr_columns"] == 32 * st["ppr_sweeps"]                          # the fp16-state solver ran
    assert 0.0 < st["ppr_residual"] < 5e-3 and st["ppr_error_bound"] < 1e-5    # and its residual check passed
    P = ppr.transition_matrix(ppr.symmetric_weights(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w))[0]
    tb = retrieve.Tables(kg.n_nodes, kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    for q in (0, 5, 11, 17, 23, 31, 32, 39):
        fs = retrieve.fact_scores(fe, qf[q])
        assert list(retrieve.top_facts(fs, 5)) == list(fidx[q]), f"query {q}: top-5 facts differ"
        np.testing.assert_allclose(fscore[q], fs[fidx[q]], atol=1e-5)
        o = retrieve.retrieve_one(P, tb, fe, pe, qf[q], qp[q], top_k=None)
        full = np.empty(len(o["ids"]))
        full[o["ids"]] = o["scores"]
        assert_topk_matches(ids[q], scores[q], full, 200, what=f"C3 d=768 query {q}")


def test_power_law_hub_shape_against_the_oracle():
    """BASELINE config #5's topology at a size the float64 oracle handles: a power-law KG whose heaviest entity has
    degree > 1e5 (rows that long are cut into 256-non-zero segments: k_sweep_long_segments + the fixed-order
    finalize), fp32 and fp16-state solvers, streamed (bf16-planes-only) fact upload."""
    import hipporag_b200 as hb
    from hipporag_b200 import synth
    kg = synth.make_kg(300_000, 3_000_000, seed=5, topology="powerlaw", zipf_q=0.5)
    deg = np.bincount(np.concatenate([kg.edge_src, kg.edge_dst]), minlength=kg.n_nodes)
    assert deg.max() > 100_000
    d = 64
    fe = synth.unit_rows(kg.n_facts, d, seed=1)
    pe = synth.unit_rows(kg.n_pass, d, seed=2)
    qf, qp, planted = synth.make_queries(kg, fe, pe, 40, seed=3)
    e = hb.Engine(0)
    e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    step = 100_000                                                             # streamed: chunks, no fp32 copy kept
    e.load_embeddings_streamed(0, kg.n_facts, d, ((lo, fe[lo:lo + step]) for lo in range(0, kg.n_facts, step)))
    e.load_embeddings_streamed(1, kg.n_pass, d, [(0, pe)])
    P = ppr.transition_matrix(ppr.symmetric_weights(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w))[0]
    tb = retrieve.Tables(kg.n_nodes, kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    for nq in (40, 6):                                                         # 40 -> fp16-state solver, 6 -> fp32
        idx, score, nv = e.stage_a(qf[:nq], 5)
        ids, scores = e.stage_b(qp[:nq], idx, score, topk=100)
        st = e.stats()
        for q in (0, nq // 2, nq - 1):
            o = retrieve.retrieve_one(P, tb, fe, pe, qf[q], qp[q], top_k=None)
            assert list(o["facts"]) == list(idx[q])
            full = np.empty(len(o["ids"]))
            full[o["ids"]] = o["scores"]
            assert_topk_matches(ids[q], scores[q], full, 100, what=f"power-law hub, {nq} queries, query {q}")
    with pytest.raises(hb.HragError, match="fp32 embedding matrix was not kept"):
        e.set_options(sim_mode=hb.SIM_FP32)
        e.stage_a(qf[:2], 5)
