"""The first solve of each stage-B sub-batch reads its first iterate x0 = rhs compactly: sweep 1 gathers rhs[slot_map[c]]
and skips the columns without a slot, sweep 2 takes prev from the rhs row.  Engine.debug_dense_first_sweep forces the
dense first iterate (scattered into [N, 32] / [N, 2, 32] and swept like any other iterate); both forms must give the
same ids, scores and stats bit for bit on one handle, and stage B must still equal hrag_ppr on the same reset."""
import numpy as np
import pytest

from tests.test_gpu_ppr_exact import StageB, exact_graph
from tests.test_gpu_ppr_paired import _check_stage_b

STATS = ("ppr_sweeps", "ppr_columns", "ppr_residual")


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def _both(e, run):
    """run() with the compact first iterate and then with the dense one: (compact result, stats), (dense ...)"""
    out = []
    for dense in (False, True):
        e.debug_dense_first_sweep(dense)
        try:
            e.reset_stats()
            r = run()
            st = e.stats()
        finally:
            e.debug_dense_first_sweep(False)
        out.append((r, {k: st[k] for k in STATS}))
    return out


def _assert_bits(a, b, what):
    for x, y in zip(a, b):
        x, y = np.asarray(x), np.asarray(y)
        assert x.dtype == y.dtype and x.shape == y.shape, what
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), what


def _compare_stage_b(s, Qi, kept, ks, iters, what, dpr_only=None):
    q = (Qi / 4).astype(np.float32)

    def run():
        return s.e.stage_b(q, kept, ks, dpr_only=dpr_only, passage_node_weight=0.5, link_top_k=10, topk=s.P,
                           iters=iters)
    (got, st), (want, st_dense) = _both(s.e, run)
    _assert_bits(got, want, what)
    assert st == st_dense, (what, st, st_dense)
    assert st["ppr_sweeps"] > 0, what
    return got


def _stage_b_on(hb, g):
    """StageB's tables and embeddings over the CSR graph g (power-of-two values, exact sums)."""
    s = StageB.__new__(StageB)
    ref = StageB(hb)
    s.__dict__.update({k: v for k, v in ref.__dict__.items() if k != "e"})
    ref.e.close()
    s.kg = type("KG", (), {"n_nodes": g.n})()
    rng = np.random.default_rng(5)
    s.passage_vid = rng.choice(g.n, s.P, replace=False).astype(np.int32)
    ents = np.setdiff1d(np.arange(g.n), s.passage_vid)
    s.subj = rng.choice(ents, s.F).astype(np.int32)
    s.obj = rng.choice(ents, s.F).astype(np.int32)
    s.subj[5] = s.passage_vid[7]                              # a seed on a passage vertex
    s.cc = (2 ** rng.integers(0, 3, g.n)).astype(np.int32)
    s.e = hb.Engine(0)
    s.e.load_graph_csr(g.n, g.row_ptr, g.col, g.val)
    s.e.load_tables(s.passage_vid, s.subj, s.obj, s.cc)
    s.e.load_embeddings(np.ones((s.F, 8), np.float32), (s.Ep / 4).astype(np.float32))
    return s


@pytest.mark.gpu
def test_first_sweep_musique1k(hb, golden):
    """C1: 64 queries, one pair per call, on the real graph; plus the odd sub-batch of 96 queries."""
    g = golden
    r = hb.B200Retriever(int(g["n_nodes"]), g["edge_src"], g["edge_dst"], g["edge_w"], g["passage_vid"],
                         g["fact_subj_vid"], g["fact_obj_vid"], g["ent_chunk_count"], g["fact_emb"],
                         g["passage_emb"], damping=float(g["damping"]), linking_top_k=int(g["linking_top_k"]),
                         passage_node_weight=float(g["passage_node_weight"]), retrieval_top_k=int(g["topk"]))
    try:
        r.engine.set_options(ppr_precision=hb.PPR_MIXED)
        for B in (64, 96):
            sel = np.arange(B) % len(g["q_fact"])
            qf, qp = g["q_fact"][sel], g["q_pass"][sel]
            (got, st), (want, st_dense) = _both(r.engine, lambda: r.retrieve(qf, qp, topk=200)[:2])
            _assert_bits(got, want, f"C1, {B} queries")
            assert st == st_dense and st["ppr_columns"] >= 64, (st, st_dense)
    finally:
        r.engine.close()


@pytest.mark.gpu
def test_first_sweep_long_rows_and_hub(hb):
    """Rows of 255 / 256 / 257 / 513 non-zeros and a hub of 2,000 (long-row segments and finalize, in pairs and in the
    odd single sub-batch); seeds on and off passage vertices, different in every query; both against hrag_ppr."""
    g = exact_graph(3000, 13, extra_lengths=(255, 256, 257, 513, 2000))
    assert {255, 256, 257, 513, 2000} <= set(np.diff(g.row_ptr).tolist())
    s = _stage_b_on(hb, g)
    try:
        for B, seed in ((64, 1), (133, 2), (33, 3)):
            Qi, kept, ks = s.queries(B, seed)
            for iters in (1, 2, 0):
                what = f"long rows, B={B} iters={iters}"
                _compare_stage_b(s, Qi, kept, ks, iters, what)
                _check_stage_b(s, Qi, kept, ks, iters, what)
    finally:
        s.e.close()


@pytest.mark.gpu
def test_first_sweep_dpr_rows_and_replay(hb):
    """DPR-fallback queries mixed into the pairs; a second call replays the captured solves, and after the tables are
    reloaded (invalidate_solves: slot maps rebuilt, graphs dropped) a fresh capture gives the same bytes."""
    s = StageB(hb)
    try:
        Qi, kept, ks = s.queries(133, 7)
        dpr = np.zeros(133, bool)
        dpr[[0, 31, 32, 70, 132]] = True
        first = _compare_stage_b(s, Qi, kept, ks, 0, "dpr rows", dpr_only=dpr)
        _assert_bits(_compare_stage_b(s, Qi, kept, ks, 0, "replayed", dpr_only=dpr), first, "replayed")
        s.e.load_tables(s.passage_vid, s.subj, s.obj, s.cc)
        _assert_bits(_compare_stage_b(s, Qi, kept, ks, 0, "after reload", dpr_only=dpr), first, "after reload")
        _check_stage_b(s, Qi[~dpr], kept[~dpr], ks[~dpr], 0, "stage B vs hrag_ppr")
    finally:
        s.e.close()


@pytest.mark.gpu
def test_first_sweep_retrieve_resident():
    """retrieve_resident over three chunks (the next chunk's similarity overlapped with the sweeps)."""
    import torch
    import hipporag_b200 as hb
    from hipporag_b200 import synth
    from tests.test_gpu_resident_pipeline import DIM, _resident
    kg = synth.make_kg(4000, 40000, seed=12)
    fe = synth.unit_rows(kg.n_facts, DIM, seed=1)
    pe = synth.unit_rows(kg.n_pass, DIM, seed=2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 2100, seed=8)
    e = hb.Engine(0)
    try:
        e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
        e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        e.load_embeddings(fe, pe)
        dqf, dqp = torch.from_numpy(qf).cuda(), torch.from_numpy(qp).cuda()
        (got, st), (want, st_dense) = _both(e, lambda: _resident(e, dqf, dqp))
        _assert_bits(got, want, "retrieve_resident")
        assert st == st_dense, (st, st_dense)
    finally:
        e.close()
