"""Fact planes in pinned host memory (hrag_set_fact_memory): a handle whose fact planes exceed its device budget keeps
them on the host and streams them through a two-slice device ring.  Every entry must return, byte for byte, what a
resident handle returns for the same inputs; the budget must hold; the entries that need resident planes must refuse
cleanly and leave the handle as it was.

A ring of two slices fits inside a budget below the planes only when a slice is less than half the fact rows, so host
planes always stream at least three slices; budgets that would give one or two slices (or cover no facts at all)
leave the planes resident, and are checked here to do exactly that.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIM = 64
SIM_BF16X3, SIM_BF16 = 1, 2
KS = (1, 5, 8, 9, 16, 32)


def _ring_budget(slice_rows, dim=DIM, slack=1000):
    """A budget whose ring holds two slices of slice_rows rows (the slack is rounded away)."""
    return 2 * slice_rows * dim * 4 + slack


def _ceil256(x):
    return -(-int(x) // 256) * 256


@pytest.fixture(scope="module")
def world():
    import torch
    import hipporag_b200 as hb
    from hipporag_b200 import synth
    kg = synth.make_kg(3000, 30000, seed=21)
    F = kg.n_facts
    assert F % 256 != 0
    fe = synth.unit_rows(F, DIM, seed=1)
    pe = synth.unit_rows(kg.n_pass, DIM, seed=2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 1300, seed=5)     # two chunks of retrieve_resident

    def engine(budget=0, emb=None):
        e = hb.Engine(0, fact_device_bytes=budget)
        e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
        e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        e.load_embeddings(fe if emb is None else emb, pe)
        return e

    budgets = {
        "3 slices": _ring_budget(_ceil256(F / 3)),
        "4 slices": _ring_budget(_ceil256(F / 4)),
        "256-row slices": _ring_budget(256),
        "planes exactly": F * DIM * 4,          # resident
        "no limit": 0,                          # resident
    }
    engines = {name: engine(b) for name, b in budgets.items()}
    ref = engine()
    yield dict(kg=kg, F=F, fe=fe, pe=pe, qf=qf, qp=qp, engines=engines, budgets=budgets, ref=ref, engine=engine,
               dqf=torch.from_numpy(qf).cuda(), dqp=torch.from_numpy(qp).cuda())
    for e in engines.values():
        e.close()
    ref.close()


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    assert got.tobytes() == want.tobytes(), f"{what}: {int((got != want).sum())} entries differ"


def _set_mode(engines, mode, keep):
    for e in engines:
        e.set_options(sim_mode=mode)
        e.debug_keep_scores(keep)


BUDGETS = ["3 slices", "4 slices", "256-row slices", "planes exactly", "no limit"]


@pytest.mark.parametrize("budget", BUDGETS)
def test_placement_and_budget(world, budget):
    e, F, b = world["engines"][budget], world["F"], world["budgets"][budget]
    info = e.fact_planes_info()
    if b and b < F * DIM * 4:
        S = (b // (2 * DIM * 4)) // 256 * 256
        assert info == {"on_host": 1, "slice_rows": S, "device_bytes": 2 * S * DIM * 4, "host_bytes": F * DIM * 4}
        assert info["device_bytes"] <= b and -(-F // S) >= 3
    else:
        assert info == {"on_host": 0, "slice_rows": 0, "device_bytes": F * DIM * 4, "host_bytes": 0}


@pytest.mark.parametrize("keep", [False, True])
@pytest.mark.parametrize("mode", [SIM_BF16X3, SIM_BF16])
@pytest.mark.parametrize("budget", BUDGETS)
def test_stage_a_and_similarity_equal_resident(world, budget, mode, keep):
    e, ref = world["engines"][budget], world["ref"]
    q = world["qf"][:300]
    _set_mode((e, ref), mode, keep)
    try:
        for k in KS:
            got, want = e.stage_a(q, k), ref.stage_a(q, k)
            for g, w, name in zip(got, want, ("ids", "scores", "n_valid")):
                _same(g, w, f"stage_a k={k} {name}")
        _same(e.similarity(0, q[:40]), ref.similarity(0, q[:40]), "similarity(0)")
        for k in (1, 32, 300):
            for g, w in zip(e.topk_similarity(0, q[:40], k), ref.topk_similarity(0, q[:40], k)):
                _same(g, w, f"topk_similarity(0) k={k}")
    finally:
        _set_mode((e, ref), SIM_BF16X3, False)


@pytest.mark.parametrize("link_top_k", [5, 16])
@pytest.mark.parametrize("mode", [SIM_BF16X3, SIM_BF16])
@pytest.mark.parametrize("budget", ["3 slices", "256-row slices"])
def test_retrieve_resident_equals_resident(world, budget, mode, link_top_k):
    import torch
    e, ref = world["engines"][budget], world["ref"]
    dqf, dqp = world["dqf"], world["dqp"]
    B = dqf.shape[0]
    outs = []
    _set_mode((e, ref), mode, False)
    try:
        for eng in (e, ref):
            oi = torch.empty((B, 50), dtype=torch.int32, device="cuda")
            os_ = torch.empty((B, 50), dtype=torch.float32, device="cuda")
            eng.retrieve_resident(dqf, dqp, oi, os_, link_top_k=link_top_k, topk=50)
            torch.cuda.synchronize()
            outs.append((oi.cpu().numpy(), os_.cpu().numpy()))
    finally:
        _set_mode((e, ref), SIM_BF16X3, False)
    _same(outs[0][0], outs[1][0], "retrieve_resident ids")
    _same(outs[0][1], outs[1][1], "retrieve_resident scores")


def test_planes_equal_resident_planes(world):
    import torch
    e, ref = world["engines"]["3 slices"], world["ref"]
    for plane in ("fact_hi", "fact_lo"):
        _same(e.debug_index(plane), ref.debug_index(plane), plane)
    assert e.debug_index("fact_f32", size_only=True) == 0
    # the streamed loader, fed device chunks, fills the same host planes
    import hipporag_b200 as hb
    s = hb.Engine(0, fact_device_bytes=world["budgets"]["4 slices"])
    try:
        fe = torch.from_numpy(world["fe"]).cuda()
        F = world["F"]
        s.load_embeddings_streamed(0, F, DIM, ((r, fe[r:r + 1000].contiguous()) for r in range(0, F, 1000)))
        assert s.fact_planes_info()["on_host"] == 1
        for plane in ("fact_hi", "fact_lo"):
            _same(s.debug_index(plane), ref.debug_index(plane), f"streamed load {plane}")
    finally:
        s.close()


@pytest.mark.parametrize("mode", [SIM_BF16X3, SIM_BF16])
def test_one_pass_per_call(world, mode):
    e, F = world["engines"]["4 slices"], world["F"]
    q = np.ascontiguousarray(np.tile(world["qf"], (3, 1))[:3000])
    e.set_options(sim_mode=mode)
    try:
        e.reset_stats()
        e.stage_a(q, 5)
        h2d = e.stats()["h2d_bytes"]
    finally:
        e.set_options(sim_mode=SIM_BF16X3)
    planes = F * DIM * 2 * (2 if mode == SIM_BF16X3 else 1)
    assert h2d == planes + q.nbytes


def test_rejections_leave_the_handle_unchanged(world):
    import torch
    import hipporag_b200 as hb
    from hipporag_b200 import HragError
    kg, fe, pe, F = world["kg"], world["fe"], world["pe"], world["F"]
    q = world["qf"][:64]
    e = hb.Engine(0, mutable=True, fact_device_bytes=world["budgets"]["3 slices"])
    try:
        e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
        e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        e.load_embeddings(fe, pe)
        want = e.stage_a(q, 5)
        with pytest.raises(HragError, match="hrag_knn_threshold: the fact planes are held in host memory"):
            e.knn_threshold(0, q, 0.5)
        with pytest.raises(HragError, match="hrag_index_reserve: the fact planes are held in host memory"):
            e.reserve(facts=F + 10)
        with pytest.raises(HragError, match="hrag_index_append: the fact planes are held in host memory"):
            e.append(0, ent_chunk_count=kg.ent_chunk_count)
        with pytest.raises(HragError, match="hrag_index_delete: the fact planes are held in host memory"):
            e.delete(facts=[0], ent_chunk_count=kg.ent_chunk_count)
        with pytest.raises(HragError, match="pass the fp32 fact rows from host memory"):
            e.load_embeddings(torch.from_numpy(fe).cuda(), pe)
        e.set_options(sim_mode=0)
        with pytest.raises(HragError, match="only the tensor-core modes are available"):
            e.stage_a(q, 5)
        e.set_options(sim_mode=SIM_BF16X3)
        for g, w in zip(e.stage_a(q, 5), want):
            _same(g, w, "stage_a after the rejections")
        assert e.fact_planes_info()["on_host"] == 1
        # a budget below two 256-row slices fails the load with its reason
        e.set_fact_memory(2 * 256 * DIM * 4 - 1)
        with pytest.raises(HragError, match="ring of two 256-row slices"):
            e.load_embeddings(fe, pe)
    finally:
        e.close()


def test_no_facts(world):
    import hipporag_b200 as hb
    pe, q = world["pe"], world["qf"][:16]
    out = []
    for budget in (0, _ring_budget(256)):
        e = hb.Engine(0, fact_device_bytes=budget)
        try:
            e.load_embeddings(np.zeros((0, DIM), np.float32), pe)
            assert e.fact_planes_info()["on_host"] == 0
            out.append(e.stage_a(q, 8))
        finally:
            e.close()
    for g, w in zip(*out):
        _same(g, w, "stage_a without facts")


# ------------------------------------------------------------------------------ exact scores across slice edges
def test_exact_ties_and_minmax_across_slice_edges():
    """Embeddings of small integers / 4: every score is exact in every mode, so ties are real.  Rows S - 1 and S tie
    for the best score of query 0 (the lower row first); 300 rows straddling S tie for query 1 (k = 32 keeps the 32
    lowest); query 2's min and max come from the first and third slice."""
    import hipporag_b200 as hb
    from tests.test_gpu_selection_exact import as_f32, exact_ints, expected_topk, minmax32, raw_scores, ranking
    rng = np.random.default_rng(3)
    S, F = 256, 3 * 256 + 100
    Ei = exact_ints(rng, (F, DIM), -2, 2)
    Ei[S - 1, 0:16] = Ei[S, 0:16] = 3
    Ei[S - 150:S + 150, 16:32] = 3
    Ei[7, 32:48], Ei[2 * S + 11, 32:48] = -3, 3
    Qi = np.zeros((3, DIM), np.int64)
    Qi[0, 0:16], Qi[1, 16:32], Qi[2, 32:48] = 3, 3, 3
    E, Q = as_f32(Ei), as_f32(Qi)
    P = as_f32(exact_ints(rng, (40, DIM)))
    raw = raw_scores(Qi, Ei)
    assert raw[0, S - 1] == raw[0, S] == raw[0].max() and (raw[0] == raw[0].max()).sum() == 2
    assert (raw[1] == raw[1].max()).sum() == 300
    assert raw[2].argmin() == 7 and raw[2].argmax() == 2 * S + 11
    host = hb.Engine(0, fact_device_bytes=_ring_budget(S))
    ref = hb.Engine(0)
    try:
        for e in (host, ref):
            e.load_embeddings(E, P)
        assert host.fact_planes_info()["slice_rows"] == S
        order = ranking(raw)
        norm = minmax32(raw)
        for mode in (SIM_BF16X3, SIM_BF16):
            for keep in (False, True):
                _set_mode((host, ref), mode, keep)
                for k in (2, 8, 9, 32):
                    ids, sc, nv = host.stage_a(Q, k)
                    wi, ws, wn = expected_topk(norm, order, k)
                    _same(ids, wi, f"ids k={k} mode={mode}")
                    _same(sc, ws, f"scores k={k} mode={mode}")
                    _same(nv, wn, f"n_valid k={k}")
                    for g, w in zip((ids, sc, nv), ref.stage_a(Q, k)):
                        _same(g, w, f"resident k={k} mode={mode}")
                assert list(ids[0, :2]) == [S - 1, S]
                assert list(ids[1]) == list(range(S - 150, S - 150 + 32))
                ti, ts = host.topk_similarity(0, Q, 32)
                wi, ws, _ = expected_topk(raw, order, 32)
                _same(ti, wi, "topk_similarity ids")
                _same(ts, ws, "topk_similarity scores")
                _same(host.similarity(0, Q), norm, "similarity")
    finally:
        host.close()
        ref.close()


# ------------------------------------------------------------------------------ the drop-in
def test_accelerate_with_a_fact_budget_equals_resident(golden):
    from tests import fake_hipporag
    fake_hipporag.install_stub_package()
    import hipporag_b200
    from hipporag_b200 import synth
    g = golden
    n, P = int(g["n_nodes"]), int(g["passage_vid"].shape[0])
    kg = synth.SynthKG(n_nodes=n, n_ent=n - P, n_pass=P, edge_src=g["edge_src"], edge_dst=g["edge_dst"],
                       edge_w=g["edge_w"], passage_vid=g["passage_vid"], fact_subj_vid=g["fact_subj_vid"],
                       fact_obj_vid=g["fact_obj_vid"], ent_chunk_count=g["ent_chunk_count"],
                       fact_passage=np.zeros(g["fact_subj_vid"].shape[0], np.int32))
    queries = [f"question {i}" for i in range(g["q_fact"].shape[0])]
    dim = int(g["dim"])
    sols = []
    for budget in (None, _ring_budget(1024, dim)):
        rag = fake_hipporag.FakeRag(kg, g["fact_emb"], g["passage_emb"], g["q_fact"], g["q_pass"], queries)
        hipporag_b200.accelerate(rag, device=0, cache=False, fact_device_bytes=budget)
        sols.append(rag.retrieve(queries, num_to_retrieve=50))
        eng = rag._b200_state["engine"]
        assert eng.fact_planes_info()["on_host"] == (0 if budget is None else 1)
        eng.close()
    for a, b in zip(*sols):
        assert a.docs == b.docs
        _same(a.doc_scores, b.doc_scores, "doc_scores")
