"""hrag_stage_b_f64 (stage B at PRPACK accuracy: the float64 reset built on the device, float64 PPR by iterative
refinement, float64 gather and exact top-k) against float64 oracles built from the engine's own fp32 inputs:
MuSiQue-1k, a reset fp32 cannot hold, the DPR fallback, ties and edges, batching, a long-row hub, the call contract,
and accelerate(run_ppr_fp64=True).retrieve."""
import numpy as np
import pytest

from oracle import ppr, prpack_gs
from tests.test_gpu_ppr_f64 import _l1, _order_ok, _powerlaw_graph

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def host_reset(n, passage_vid, fact_subj, fact_obj, chunk_count, kept_idx, kept_score, pass_norm, link_top_k=5,
               pnw=0.05):
    """graph_search_with_fact_entities' node_weights in the reference's dtypes (HippoRAG.py:1583-1638): phrase weight
    float32(score) / float32(chunk count) accumulated and averaged in float64, the link_top_k best phrases kept (tie ->
    lower vertex); passage weight float32(minmax score) * float32(pnw) stored as float64; their float64 sum."""
    phrase = np.zeros(n)
    occ = np.zeros(n)
    touched = []
    for f, s in zip(kept_idx, kept_score):
        if f < 0:
            continue
        for v in (int(fact_subj[f]), int(fact_obj[f])):
            if v < 0:
                continue
            w = np.float32(s)
            if chunk_count[v] > 0:
                w = np.float32(s) / np.float32(chunk_count[v])
            phrase[v] += np.float64(w)
            occ[v] += 1
            if v not in touched:
                touched.append(v)
    nz = occ > 0
    phrase[nz] /= occ[nz]
    if link_top_k:
        keep = sorted(touched, key=lambda v: (-phrase[v], v))[:link_top_k]
        mask = np.zeros(n, bool)
        mask[keep] = True
        phrase[~mask] = 0.0
    passage = np.zeros(n)
    passage[passage_vid] = (np.asarray(pass_norm, np.float32) * np.float32(pnw)).astype(np.float64)
    return phrase + passage


def resets_for(e, tables, kept_idx, kept_score, q_pass, link_top_k=5, pnw=0.05):
    sim = e.similarity(1, q_pass)                       # the GEMM + min-max the device reset reads
    n, pv, fs, fo, cc = tables
    return np.stack([host_reset(n, pv, fs, fo, cc, kept_idx[q], kept_score[q], sim[q], link_top_k, pnw)
                     for q in range(q_pass.shape[0])])


def criterion(ids, scores, doc, tol):
    """returned scores within tol (L1) of the oracle's, the oracle's order on the window, and the oracle's top-k set
    except for pairs within 2 tol of its k-th score"""
    k = ids.shape[0]
    if not np.all(ids >= 0):
        return False
    want = np.lexsort((np.arange(doc.shape[0]), -doc))[:k]
    kth = doc[want[-1]]
    members = all(abs(doc[i] - kth) <= 2 * tol for i in set(ids.tolist()) ^ set(want.tolist()))
    return bool(_l1(scores, doc[ids]) <= tol and _order_ok(scores, doc[ids], tol) and members)


def exact_order(ids, scores):
    """(score desc, id asc), strictly"""
    return bool(np.all((scores[:-1] > scores[1:]) | ((scores[:-1] == scores[1:]) & (ids[:-1] < ids[1:]))))


@pytest.fixture(scope="module")
def mq(hb, golden):
    g = golden
    e = hb.Engine(0)
    e.load_graph(int(g["n_nodes"]), g["edge_src"], g["edge_dst"], g["edge_w"])
    e.load_tables(g["passage_vid"], g["fact_subj_vid"], g["fact_obj_vid"], g["ent_chunk_count"])
    e.load_embeddings(g["fact_emb"], g["passage_emb"])
    tables = (int(g["n_nodes"]), g["passage_vid"], g["fact_subj_vid"], g["fact_obj_vid"], g["ent_chunk_count"])
    idx, score, _ = e.stage_a(g["q_fact"], int(g["linking_top_k"]))
    return e, tables, idx, score


def test_musique1k_against_sparse_lu(hb, golden, mq):
    g = golden
    e, tables, idx, score = mq
    a, pnw, ltk, k = float(g["damping"]), float(g["passage_node_weight"]), int(g["linking_top_k"]), 200
    Q = g["q_pass"].shape[0]
    R = resets_for(e, tables, idx, score, g["q_pass"], ltk, pnw)
    lu = ppr.factorize(g["P"], a)
    doc = np.stack([ppr.ppr_direct(g["P"], r, a, lu=lu)[g["passage_vid"]] for r in R])
    # premise: the DPR rows of stage B are the top-k of the same GEMM + min-max the oracle's reset reads
    sim = e.similarity(1, g["q_pass"])
    ids_d, sc_d = e.stage_b_f64(g["q_pass"], idx, score, np.ones(Q, np.uint8), a, pnw, ltk, k)
    for q in range(Q):
        o = np.lexsort((np.arange(sim.shape[1]), -sim[q]))[:k]
        assert np.array_equal(ids_d[q], o)
        assert sc_d[q].tobytes() == sim[q, o].astype(np.float64).tobytes()
    for tol in (0.0, 1e-12):
        want = tol or 1e-10
        ids, scores = e.stage_b_f64(g["q_pass"], idx, score, None, a, pnw, ltk, k, tol=tol)
        assert ids.dtype == np.int32 and scores.dtype == np.float64 and scores.shape == (Q, k)
        bad = [q for q in range(Q) if not criterion(ids[q], scores[q], doc[q], want)]
        assert not bad, (tol, bad[:5])
        assert 0.0 < e.stats()["ppr_error_bound"] <= want
    # teeth: the fp32 stage B misses the same criterion
    ids32, sc32 = e.stage_b(g["q_pass"], idx, score, None, a, pnw, ltk, k)
    assert not all(criterion(ids32[q], sc32[q].astype(np.float64), doc[q], 1e-10) for q in range(Q))


def _tiny_kg(n_pass=12):
    """4 entities (chunk counts 3, 7, 3, 7) linked to passages 4..4+n_pass; facts over the entities."""
    n_ent = 4
    n = n_ent + n_pass
    src = [0, 0, 1, 1, 2, 3, 0, 2]
    dst = [1, 4, 5, 6, 7, 8, 9, 3]
    w = [1.0, 2.0, 1.0, 1.5, 1.0, 3.0, 0.7, 1.0]
    pv = np.arange(n_ent, n, dtype=np.int32)
    fs = np.array([0, 0, 1, 2, 3], np.int32)
    fo = np.array([1, 2, 3, 3, 0], np.int32)
    cc = np.zeros(n, np.int32)
    cc[:4] = [3, 7, 3, 7]
    return n, src, dst, w, pv, fs, fo, cc


def test_reset_keeps_float64_phrase_weights(hb):
    n, src, dst, w, pv, fs, fo, cc = _tiny_kg()
    rng = np.random.default_rng(4)
    d = 64
    fe = rng.standard_normal((fs.shape[0], d)).astype(np.float32)
    pe = rng.standard_normal((pv.shape[0], d)).astype(np.float32)
    qf = rng.standard_normal((3, d)).astype(np.float32)
    qp = rng.standard_normal((3, d)).astype(np.float32)
    e = hb.Engine(0)
    e.load_graph(n, src, dst, w)
    e.load_tables(pv, fs, fo, cc)
    e.load_embeddings(fe, pe)
    idx, score, _ = e.stage_a(qf, 5)
    R = resets_for(e, (n, pv, fs, fo, cc), idx, score, qp)
    # the mean phrase weights of these resets are not fp32 numbers
    assert np.any(R != R.astype(np.float32).astype(np.float64))
    P = ppr.transition_matrix(ppr.symmetric_weights(n, src, dst, w))[0]
    ids, scores = e.stage_b_f64(qp, idx, score, topk=pv.shape[0], tol=1e-12)
    R32 = R.astype(np.float32).astype(np.float64)
    for q in range(3):
        doc = ppr.ppr_direct(P, R[q], 0.5)[pv]
        assert _l1(scores[q], doc[ids[q]]) <= 1e-12, _l1(scores[q], doc[ids[q]])
        # seed weights rounded to fp32 (what the fp32 stage B stores) move the result by far more than the target
        assert _l1(ppr.ppr_direct(P, R32[q], 0.5)[pv], doc) > 1e-11


def test_dpr_fallback_is_stage_b_widened(hb, golden, mq):
    g = golden
    e, _, idx, score = mq
    Q = 6
    kept = idx[:Q].copy()
    kept[1] = -1                                 # nothing kept -> DPR
    flags = np.zeros(Q, np.uint8)
    flags[3] = 1                                 # flagged -> DPR
    ids32, sc32 = e.stage_b(g["q_pass"][:Q], kept, score[:Q], flags, topk=50)
    ids, sc = e.stage_b_f64(g["q_pass"][:Q], kept, score[:Q], flags, topk=50)
    for q in (1, 3):
        assert np.array_equal(ids[q], ids32[q])
        assert sc[q].tobytes() == sc32[q].astype(np.float64).tobytes()
    none = np.zeros((Q, 0), np.int32)            # k_facts == 0 (retrieve_dpr): every row
    ids32, sc32 = e.stage_b(g["q_pass"][:Q], none, none.astype(np.float32), topk=50)
    ids, sc = e.stage_b_f64(g["q_pass"][:Q], none, none.astype(np.float32), topk=50)
    assert np.array_equal(ids, ids32)
    assert sc.tobytes() == sc32.astype(np.float64).tobytes()


def test_ties_padding_and_deep_topk(hb):
    # passages 4..15: 9..15 are isolated; 10, 11, 13 and 14 have the query's own embedding (equal DPR scores)
    n, src, dst, w, pv, fs, fo, cc = _tiny_kg()
    rng = np.random.default_rng(8)
    d = 64
    base = rng.standard_normal((8, d)).astype(np.float32)
    base /= np.linalg.norm(base, axis=1, keepdims=True)
    pe = base[np.array([1, 2, 3, 4, 5, 6, 0, 0, 7, 0, 0, 6])]
    fe = base[np.array([1, 2, 3, 4, 5])]
    e = hb.Engine(0)
    e.load_graph(n, src, dst, w)
    e.load_tables(pv, fs, fo, cc)
    e.load_embeddings(fe, pe)
    qf, qp = base[1:2].copy(), base[0:1].copy()
    idx, score, _ = e.stage_a(qf, 5)
    ids, sc = e.stage_b_f64(qp, idx, score, topk=16)
    P = pv.shape[0]
    assert np.all(ids[0, P:] == -1) and np.all(sc[0, P:] == 0.0)
    full_ids, full = ids[0, :P], sc[0, :P]
    assert sorted(full_ids.tolist()) == list(range(P)) and exact_order(full_ids, full)
    tied = [6, 7, 9, 10]
    assert len({full[full_ids == p][0] for p in tied}) == 1             # bitwise-equal pi
    pos = int(np.flatnonzero(np.isin(full_ids, tied))[0])
    for cut in (pos + 1, pos + 2, pos + 3):                            # the cut inside the tied group
        ids_k, sc_k = e.stage_b_f64(qp, idx, score, topk=cut)
        assert np.array_equal(ids_k[0], full_ids[:cut]) and sc_k[0].tobytes() == full[:cut].tobytes()
    # topk = 2048 on more passages than that
    from hipporag_b200 import synth
    kg = synth.make_kg(30000, 150000, seed=3)
    assert kg.n_pass > 2048
    fe, pe = synth.unit_rows(kg.n_facts, 64, 1), synth.unit_rows(kg.n_pass, 64, 2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 3, seed=5)
    e = hb.Engine(0)
    e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    e.load_embeddings(fe, pe)
    idx, score, _ = e.stage_a(qf, 5)
    ids, sc = e.stage_b_f64(qp, idx, score, topk=2048)
    R = resets_for(e, (kg.n_nodes, kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count), idx,
                   score, qp)
    Pm = ppr.transition_matrix(ppr.symmetric_weights(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w))[0]
    O = ppr.ppr_batch_power(Pm, R.T, 0.5).T        # to 1e-14 (a sparse LU of this random graph fills in)
    for q in range(3):
        assert exact_order(ids[q], sc[q])
        assert criterion(ids[q], sc[q], O[q][kg.passage_vid], 1e-10)


@pytest.mark.parametrize("B", [1, 7, 16, 17, 40, 1040])
def test_batching_and_determinism(hb, golden, mq, B):
    """1040 = one full chunk of 1024 queries (MuSiQue-1k's chunk_b) and a second of 16, both 16 wide"""
    g = golden
    e, _, idx, score = mq
    rng = np.random.default_rng(B)
    sel = rng.integers(0, 64, B) if B > 64 else rng.permutation(64)[:B]
    qp, ki, ks = g["q_pass"][sel], idx[sel], score[sel]
    out = e.stage_b_f64(qp, ki, ks)
    again = e.stage_b_f64(qp, ki, ks)
    assert out[0].tobytes() == again[0].tobytes() and out[1].tobytes() == again[1].tobytes()
    perm = rng.permutation(B)
    shuf = e.stage_b_f64(qp[perm], ki[perm], ks[perm])
    assert shuf[0].tobytes() == out[0][perm].tobytes() and shuf[1].tobytes() == out[1][perm].tobytes()
    # the same query at another sub-batch width: only the summation order changes
    ids1, sc1 = e.stage_b_f64(qp[:1], ki[:1], ks[:1])
    common, i1, i0 = np.intersect1d(ids1[0], out[0][0], return_indices=True)
    assert common.shape[0] >= 190
    assert _l1(sc1[0][i1], out[1][0][i0]) <= 2e-10


@pytest.mark.parametrize("damping", [0.5, 0.85])
def test_long_rows_against_prpack_gauss_seidel(hb, damping):
    n, src, dst, w = _powerlaw_graph()
    rng = np.random.default_rng(2)
    pv = np.arange(1000, 1400, dtype=np.int32)               # passages among the power-law tail
    F = 300
    fs = rng.integers(0, 1000, F).astype(np.int32)
    fs[:20] = 0                                               # facts on the hub (a row of > 256 non-zeros)
    fo = rng.integers(0, 1000, F).astype(np.int32)
    cc = rng.integers(0, 5, n).astype(np.int32)
    d = 64
    fe = rng.standard_normal((F, d)).astype(np.float32)
    pe = rng.standard_normal((pv.shape[0], d)).astype(np.float32)
    qf = np.concatenate([fe[:2] + 0.01, rng.standard_normal((2, d)).astype(np.float32)])
    qp = rng.standard_normal((4, d)).astype(np.float32)
    e = hb.Engine(0)
    e.load_graph(n, src, dst, w)
    e.load_tables(pv, fs, fo, cc)
    e.load_embeddings(fe, pe)
    idx, score, _ = e.stage_a(qf, 5)
    ids, sc = e.stage_b_f64(qp, idx, score, damping=damping, topk=100)
    R = resets_for(e, (n, pv, fs, fo, cc), idx, score, qp)
    for q in range(4):
        want = prpack_gs.personalized_pagerank_gs(n, src, dst, w, R[q], damping)[pv]
        assert _l1(sc[q], want[ids[q]]) <= 2e-10, (q, _l1(sc[q], want[ids[q]]))
    assert e.stats()["ppr_error_bound"] <= 1e-10


def test_contract(hb, golden, mq):
    from hipporag_b200.engine import build_transition_csr
    g = golden
    e, _, idx, score = mq
    qp = g["q_pass"][:2]
    with pytest.raises(hb.HragError, match="1e-13"):
        e.stage_b_f64(qp, idx[:2], score[:2], tol=5e-14)
    for topk in (0, 2049):
        with pytest.raises(hb.HragError, match="bad sizes"):
            e.stage_b_f64(qp, idx[:2], score[:2], topk=topk)
    with pytest.raises(hb.HragError, match="bad sizes"):
        e.stage_b_f64(qp, np.zeros((2, 33), np.int32), np.zeros((2, 33), np.float32))
    for a in (0.0, 1.0, 1.5):
        with pytest.raises(hb.HragError, match="damping"):
            e.stage_b_f64(qp, idx[:2], score[:2], damping=a)
    n = int(g["n_nodes"])
    e32 = hb.Engine(0)
    e32.load_graph_csr(n, *build_transition_csr(n, g["edge_src"], g["edge_dst"], g["edge_w"]))
    e32.load_tables(g["passage_vid"], g["fact_subj_vid"], g["fact_obj_vid"], g["ent_chunk_count"])
    e32.load_embeddings(g["fact_emb"], g["passage_emb"])
    with pytest.raises(hb.HragError, match="hrag_load_graph_csr_f64 or hrag_load_graph_coo"):
        e32.stage_b_f64(qp, idx[:2], score[:2])


def test_sharded_handle_rejects(hb):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("a world > 1 handle needs two GPUs")
    import multiprocessing as mp
    with mp.get_context("spawn").Pool(2) as pool:
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
        e.stage_b_f64(np.zeros((1, 8), np.float32), np.zeros((1, 1), np.int32), np.zeros((1, 1), np.float32))
    except hb.HragError as ex:
        return str(ex)
    return "no error"


def test_accelerate_retrieve_fp64(hb):
    from tests import fake_hipporag
    from hipporag_b200 import synth
    fake_hipporag.install_stub_package()
    kg = synth.make_kg(3000, 30000, seed=5)
    fe, pe = synth.unit_rows(kg.n_facts, 64, 1), synth.unit_rows(kg.n_pass, 64, 2)
    nq = 6
    qf, qp, _ = synth.make_queries(kg, fe, pe, nq, seed=3)
    names = [f"q{i}" for i in range(nq)]
    rag = fake_hipporag.FakeRag(kg, fe, pe, qf, qp, names)
    hb.accelerate(rag, device=0, run_ppr_fp64=True)
    res = rag.retrieve(names)
    eng = rag._b200_state["engine"]
    idx, score, _ = eng.stage_a(qf, 5)
    ids, sc = eng.stage_b_f64(qp, idx, score, topk=200)
    tables = (kg.n_nodes, kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    R = resets_for(eng, tables, idx, score, qp)
    tol = 1e-10
    for q, r in enumerate(res):
        got = np.array([int(d.split()[1]) for d in r.docs])
        assert np.asarray(r.doc_scores).dtype == np.float64
        assert np.array_equal(got, ids[q]) and np.asarray(r.doc_scores).tobytes() == sc[q].tobytes()
        # the serial path: the same reset through the fp64 run_ppr drop-in
        order, full = rag.run_ppr(R[q], 0.5)
        doc = np.empty_like(full)
        doc[order] = full
        assert _l1(sc[q], doc[ids[q]]) <= tol
        gap = np.abs(np.diff(full[:201]))
        sep = (np.concatenate([[np.inf], gap[:199]]) > 2 * tol) & (gap[:200] > 2 * tol)
        assert np.array_equal(ids[q][sep], order[:200][sep])
    # the default mode is the fp32 stage B
    rag32 = fake_hipporag.FakeRag(kg, fe, pe, qf, qp, names)
    hb.accelerate(rag32, device=0)
    res32 = rag32.retrieve(names)
    e32 = rag32._b200_state["engine"]
    ids32, sc32 = e32.stage_b(qp, *e32.stage_a(qf, 5)[:2], topk=200)
    for q, r in enumerate(res32):
        assert np.array_equal([int(d.split()[1]) for d in r.docs], ids32[q])
        assert np.asarray(r.doc_scores).tobytes() == sc32[q].astype(np.float64).tobytes()
