"""Paired mixed solves: on one GPU, stage B solves consecutive 32-query sub-batches two at a time, one walk of each
row's non-zeros per sweep for both (k_sweep_h2 over [N, 2, 32] state).  hrag_ppr's dense path solves one sub-batch at
a time (k_sweep_h), so stage B must equal hrag_ppr(reset)[:, passage_vid] bit for bit and count the same sweeps."""
import numpy as np
import pytest

from tests.test_gpu_ppr_exact import StageB, assert_same, exact_graph


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


@pytest.fixture(scope="module")
def sb(hb):
    s = StageB(hb)
    yield s
    s.e.close()


def _check_stage_b(sb, Qi, kept, ks, iters, what):
    B = len(Qi)
    sb.e.reset_stats()
    got = sb.stage_b(Qi, kept, ks, iters)
    st = sb.e.stats()
    R = sb.reset(Qi, kept, ks)
    sb.e.reset_stats()
    want = sb.e.ppr(R, iters=iters)[:, sb.passage_vid]
    st_dense = sb.e.stats()
    assert st["ppr_columns"] == 32 * st["ppr_sweeps"], what
    assert st["ppr_sweeps"] == st_dense["ppr_sweeps"], what          # a pair counts as two 32-column sweeps
    assert st["ppr_sweeps"] % ((B + 31) // 32) == 0, what
    assert_same(got, want, what)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("B", [33, 40, 64, 133, 1057])
def test_paired_stage_b_equals_dense_ppr(hb, sb, B):
    """33 and 40: one pair whose partner has nb < 32; 64: one full pair; 133: two pairs (both buffer sets) and an odd
    last sub-batch on the single path; 1057: a 1,024-query chunk of 16 pairs (the captured graph of each set replayed),
    then a chunk of 33 whose pair has a 1-query partner."""
    Qi, kept, ks = sb.queries(B, B)
    for iters in (1, 0):
        _check_stage_b(sb, Qi, kept, ks, iters, f"paired stage B vs hrag_ppr B={B} iters={iters}")


@pytest.mark.gpu
def test_paired_stage_b_replayed(hb, sb):
    """The second call replays both sets' captured pair graphs: same bytes as the first call."""
    Qi, kept, ks = sb.queries(133, 5)
    first = _check_stage_b(sb, Qi, kept, ks, 0, "paired stage B, first call")
    assert_same(sb.stage_b(Qi, kept, ks), first, "paired stage B, replayed")


def _exact_stage_b(hb, n_long_extra):
    """StageB's tables and embeddings over an exact_graph: the exact premise (exactly representable sums) of
    test_gpu_ppr_exact, and with n_long_extra long rows the long-row segment / finalize kernels in a pair."""
    g = exact_graph(3000, 11, n_long_extra=n_long_extra)
    s = StageB.__new__(StageB)
    ref = StageB(hb)
    s.__dict__.update({k: v for k, v in ref.__dict__.items() if k != "e"})
    ref.e.close()
    s.kg = type("KG", (), {"n_nodes": g.n})()
    rng = np.random.default_rng(3)
    s.passage_vid = rng.choice(g.n, s.P, replace=False).astype(np.int32)
    ents = np.setdiff1d(np.arange(g.n), s.passage_vid)
    s.subj = rng.choice(ents, s.F).astype(np.int32)
    s.obj = rng.choice(ents, s.F).astype(np.int32)
    s.subj[5] = s.passage_vid[7]
    s.cc = (2 ** rng.integers(0, 3, g.n)).astype(np.int32)
    s.e = hb.Engine(0)
    s.e.load_graph_csr(g.n, g.row_ptr, g.col, g.val)
    s.e.load_tables(s.passage_vid, s.subj, s.obj, s.cc)
    s.e.load_embeddings(np.ones((s.F, 8), np.float32), (s.Ep / 4).astype(np.float32))
    return g, s


@pytest.mark.gpu
@pytest.mark.parametrize("n_long_extra", [0, 40])
def test_paired_stage_b_exact_graph(hb, n_long_extra):
    """On the exact premise graph, and on it with rows of more than 256 non-zeros (segments summed by the single-state
    long-row kernels, once per state of the pair)."""
    g, s = _exact_stage_b(hb, n_long_extra)
    if n_long_extra:
        assert np.diff(g.row_ptr).max() > 256
    try:
        Qi, kept, ks = s.queries(100, 17)
        for iters in (1, 0):
            _check_stage_b(s, Qi, kept, ks, iters, f"paired stage B, exact graph, {n_long_extra} long rows, iters={iters}")
    finally:
        s.e.close()


@pytest.mark.gpu
def test_paired_power_law_graph(hb):
    """A power-law graph with hub rows far above 256 non-zeros."""
    from hipporag_b200 import synth
    kg = synth.make_kg(20_000, 200_000, seed=4, topology="powerlaw")
    s = StageB.__new__(StageB)
    ref = StageB(hb)
    s.__dict__.update({k: v for k, v in ref.__dict__.items() if k != "e"})
    ref.e.close()
    rng = np.random.default_rng(4)
    s.kg = kg
    s.passage_vid = np.asarray(kg.passage_vid, np.int32)[:s.P]
    ents = np.setdiff1d(np.arange(kg.n_nodes), s.passage_vid)
    s.subj = rng.choice(ents, s.F).astype(np.int32)
    s.obj = rng.choice(ents, s.F).astype(np.int32)
    s.subj[5] = s.passage_vid[7]
    s.cc = (2 ** rng.integers(0, 3, kg.n_nodes)).astype(np.int32)
    s.e = hb.Engine(0)
    s.e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    s.e.load_tables(s.passage_vid, s.subj, s.obj, s.cc)
    s.e.load_embeddings(np.ones((s.F, 8), np.float32), (s.Ep / 4).astype(np.float32))
    try:
        deg = np.bincount(np.concatenate([kg.edge_src, kg.edge_dst]), minlength=kg.n_nodes)
        assert deg.max() > 256
        Qi, kept, ks = s.queries(96, 23)
        _check_stage_b(s, Qi, kept, ks, 0, "paired stage B, power-law graph")
    finally:
        s.e.close()


@pytest.mark.gpu
def test_paired_retrieve_resident_equals_single_sub_batches():
    """hrag_retrieve_resident over three chunks (2,100 queries: pairs in every chunk, the next chunk's similarity
    overlapped) against calls of 32 queries, each one sub-batch solved alone: ids and scores bit for bit, same sweeps."""
    import torch
    from hipporag_b200 import synth
    from tests.test_gpu_resident_pipeline import DIM, _resident
    kg = synth.make_kg(4000, 40000, seed=11)
    fe = synth.unit_rows(kg.n_facts, DIM, seed=1)
    pe = synth.unit_rows(kg.n_pass, DIM, seed=2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 2100, seed=6)
    import hipporag_b200 as hb
    e = hb.Engine(0)
    try:
        e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
        e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        e.load_embeddings(fe, pe)
        dqf, dqp = torch.from_numpy(qf).cuda(), torch.from_numpy(qp).cuda()
        e.reset_stats()
        got_ids, got_scores = _resident(e, dqf, dqp)
        st = e.stats()
        ids, scores, sweeps = [], [], 0
        for q0 in range(0, len(qf), 32):
            e.reset_stats()
            i, s = _resident(e, dqf[q0:q0 + 32], dqp[q0:q0 + 32])
            ids.append(i)
            scores.append(s)
            sweeps += e.stats()["ppr_sweeps"]
        assert np.array_equal(got_ids, np.concatenate(ids)), "ids differ"
        assert np.array_equal(got_scores.view(np.uint32), np.concatenate(scores).view(np.uint32)), "scores differ"
        assert st["ppr_sweeps"] == sweeps and st["ppr_columns"] == 32 * sweeps, st
    finally:
        e.close()
