"""Fact planes split between the device and the host (hrag_set_fact_placement(HRAG_FACT_LO_ON_HOST)): over the
hrag_set_fact_memory budget the hi plane stays resident and only the lo plane goes to mapped pinned host memory.  Stage
A then runs the stage-A screen on the resident hi plane and reads only the staged candidates' lo rows over PCIe; the
routes that need every lo row stream the lo plane.  Every entry must return, byte for byte, what a resident handle
returns for the same inputs; the entries that need resident planes must refuse cleanly and leave the handle as it was.
"""
import numpy as np
import pytest

from tests.test_gpu_stage_a_screen import _aligned, _cross, _err_bound, _queries, _unit

pytestmark = pytest.mark.gpu

SIM_FP32, SIM_BF16X3, SIM_BF16 = 0, 1, 2
F_SCREEN = 65_536 + 37          # screened (>= 65,536 facts), not a multiple of the 256-fact tile


def _lo_budget(rows, dim, slices=2, slack=100):
    """hi plane + `slices` 256-row lo slices (the slack is rounded away)."""
    return rows * dim * 2 + slices * 256 * dim * 2 + slack


def _same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    assert got.tobytes() == want.tobytes(), f"{what}: {int((got != want).sum())} entries differ"


def _pair(fe, pe, budget, kg=None):
    """(lo-on-host handle, resident handle) over the same inputs."""
    import hipporag_b200 as hb
    out = []
    for lo_host in (True, False):
        e = hb.Engine(0, fact_device_bytes=budget if lo_host else 0, fact_lo_on_host=lo_host)
        if kg is not None:
            e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
            e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        e.load_embeddings(fe, pe)
        out.append(e)
    return out


def _stage_a(e, Q, k, minmax=False):
    """stage_a outputs (+ the per-query (min, max) when asked), the fallbacks and h2d bytes of the call."""
    e.reset_stats()
    out = list(e.stage_a(Q, k))
    if minmax:
        out.append(e.debug_fact_minmax())
    st = e.stats()
    return out, st["stage_a_fallbacks"], st["h2d_bytes"]


def _assert_stage_a(lo, ref, Q, k, what, minmax=False, fallbacks=0):
    got, fb, h2d = _stage_a(lo, Q, k, minmax)
    want, fb_ref, h2d_ref = _stage_a(ref, Q, k, minmax)
    for g, w, name in zip(got, want, ("ids", "scores", "n_valid", "mm_fact")):
        _same(g, w, f"{what} {name}")
    assert fb == fb_ref and (fallbacks is None or fb == fallbacks), (what, fb, fb_ref)
    return h2d - h2d_ref


# ------------------------------------------------------------------------------ placement and the loaders
DIM = 64


@pytest.fixture(scope="module")
def small():
    from hipporag_b200 import synth
    kg = synth.make_kg(3000, 30000, seed=21)
    F = kg.n_facts
    assert F % 256 != 0 and F < 65_536
    return dict(kg=kg, F=F, fe=synth.unit_rows(F, DIM, seed=1), pe=synth.unit_rows(kg.n_pass, DIM, seed=2),
                q=synth.unit_rows(200, DIM, seed=3))


@pytest.mark.parametrize("slices", [2, 3, 4, 33])
def test_placement_lo_on_host(small, slices):
    import hipporag_b200 as hb
    F, pe = F_SCREEN, small["pe"]                  # room for 33 lo slices below the planes
    fe = _unit(np.random.default_rng(slices).standard_normal((F, DIM)))
    b = _lo_budget(F, DIM, slices)
    assert b < F * DIM * 4
    e = hb.Engine(0, fact_device_bytes=b, fact_lo_on_host=True)
    try:
        e.load_embeddings(fe, pe)
        S = slices // 2 * 256
        assert e.fact_planes_info() == {"on_host": 2, "slice_rows": S, "device_bytes": F * DIM * 2 + 2 * S * DIM * 2,
                                        "host_bytes": F * DIM * 2}
        assert e.fact_planes_info()["device_bytes"] <= b
    finally:
        e.close()


def test_placement_budgets(small):
    import hipporag_b200 as hb
    from hipporag_b200 import HragError
    F, fe, pe, q = small["F"], small["fe"], small["pe"], small["q"]
    # the planes exactly: resident, as by default
    e = hb.Engine(0, fact_device_bytes=F * DIM * 4, fact_lo_on_host=True)
    try:
        e.load_embeddings(fe, pe)
        assert e.fact_planes_info() == {"on_host": 0, "slice_rows": 0, "device_bytes": F * DIM * 4, "host_bytes": 0}
    finally:
        e.close()
    # the same budget as lo on host under the default placement: both planes on the host
    e = hb.Engine(0, fact_device_bytes=_lo_budget(F, DIM))
    try:
        e.load_embeddings(fe, pe)
        assert e.fact_planes_info()["on_host"] == 1
    finally:
        e.close()
    # below hi + two 256-row lo slices: the load fails with its reason and the handle keeps its planes
    e = hb.Engine(0, fact_device_bytes=_lo_budget(F, DIM), fact_lo_on_host=True)
    try:
        e.load_embeddings(fe, pe)
        want = e.stage_a(q, 5)
        info = e.fact_planes_info()
        e.set_fact_memory(_lo_budget(F, DIM, slack=0) - 1)
        with pytest.raises(HragError, match=f"hi fact plane of {F * DIM * 2} bytes"):
            e.load_embeddings(fe, pe)
        with pytest.raises(HragError, match="hi fact plane"):
            e.load_embeddings_streamed(0, F, DIM, [(0, fe)])
        assert e.fact_planes_info() == info
        for g, w in zip(e.stage_a(q, 5), want):
            _same(g, w, "stage_a after the failed load")
    finally:
        e.close()


@pytest.mark.parametrize("loader", ["whole", "host chunks", "device chunks"])
def test_planes_equal_resident_planes(small, loader):
    import torch
    F, fe, pe, q = small["F"], small["fe"], small["pe"], small["q"]
    lo, ref = _pair(fe, pe, _lo_budget(F, DIM, 3))
    try:
        if loader != "whole":
            step = 1000                      # not a multiple of the fill's 128-row steps
            chunks = [(r, fe[r:r + step]) for r in range(0, F, step)]
            if loader == "device chunks":
                chunks = [(r, torch.from_numpy(np.ascontiguousarray(c)).cuda()) for r, c in chunks]
                torch.cuda.synchronize()
            lo.load_embeddings_streamed(0, F, DIM, chunks)
        assert lo.fact_planes_info()["on_host"] == 2
        for plane in ("fact_hi", "fact_lo"):
            _same(lo.debug_index(plane), ref.debug_index(plane), f"{loader}: {plane}")
        assert lo.debug_index("fact_f32", size_only=True) == 0
        for k in (5, 16):
            for g, w in zip(lo.stage_a(q, k), ref.stage_a(q, k)):
                _same(g, w, f"{loader}: stage_a k={k}")
    finally:
        lo.close()
        ref.close()


# ------------------------------------------------------------------------------ the screen on random unit rows
@pytest.fixture(scope="module", params=[768, 1024])
def screen(request):
    dim = request.param
    rng = np.random.default_rng(dim)
    fe = _unit(rng.standard_normal((F_SCREEN, dim)))
    pe = _unit(rng.standard_normal((4, dim)))
    lo, ref = _pair(fe, pe, _lo_budget(F_SCREEN, dim))
    assert lo.fact_planes_info()["on_host"] == 2
    yield dict(dim=dim, fe=fe, lo=lo, ref=ref, rng=rng)
    lo.close()
    ref.close()


@pytest.mark.parametrize("B", [1, 1000, 1024, 2500])
def test_screen_random_unit_vectors(screen, B):
    dim, lo, ref = screen["dim"], screen["lo"], screen["ref"]
    Q = _queries(screen["fe"], B, np.random.default_rng(dim + B))
    try:
        for n_ctas in (0, 7, 61):
            lo.debug_sim_ctas(n_ctas)
            ref.debug_sim_ctas(n_ctas)
            for k in range(1, 9):
                extra = _assert_stage_a(lo, ref, Q, k, f"dim={dim} B={B} ctas={n_ctas} k={k}", minmax=B <= 1024)
                if B == 1:      # the gathered lo rows only, not a stream of the lo plane
                    assert 0 < extra < F_SCREEN * dim * 2, extra
    finally:
        lo.debug_sim_ctas(0)
        ref.debug_sim_ctas(0)


def test_unscreened_routes(screen):
    """k > 8, kept scores, the exact stage A and the similarity entries stream the lo plane; HRAG_SIM_BF16 reads the
    resident hi plane only."""
    dim, lo, ref = screen["dim"], screen["lo"], screen["ref"]
    Q = _queries(screen["fe"], 300, np.random.default_rng(7))
    for k in (9, 16, 32):
        extra = _assert_stage_a(lo, ref, Q, k, f"k={k}")
        assert extra >= F_SCREEN * dim * 2          # the whole lo plane streamed once
    for e in (lo, ref):
        e.debug_keep_scores(True)
    try:
        _assert_stage_a(lo, ref, Q, 5, "debug_keep_scores")
    finally:
        for e in (lo, ref):
            e.debug_keep_scores(False)
    for e in (lo, ref):
        e.debug_exact_stage_a(True)
    try:
        _assert_stage_a(lo, ref, Q, 5, "debug_exact_stage_a")
    finally:
        for e in (lo, ref):
            e.debug_exact_stage_a(False)
    _same(lo.similarity(0, Q[:40]), ref.similarity(0, Q[:40]), "similarity(0)")
    for k in (1, 32, 300):
        for g, w in zip(lo.topk_similarity(0, Q[:40], k), ref.topk_similarity(0, Q[:40], k)):
            _same(g, w, f"topk_similarity(0) k={k}")
    for e in (lo, ref):
        e.set_options(sim_mode=SIM_BF16)
    try:
        for k in (5, 16):
            extra = _assert_stage_a(lo, ref, Q, k, f"HRAG_SIM_BF16 k={k}")
            assert extra == 0, extra
        _same(lo.similarity(0, Q[:40]), ref.similarity(0, Q[:40]), "HRAG_SIM_BF16 similarity(0)")
    finally:
        for e in (lo, ref):
            e.set_options(sim_mode=SIM_BF16X3)


def test_below_screen_size(golden):
    """The MuSiQue-1k facts (10,734, below the screen's 65,536): every route streams the lo plane."""
    g = golden
    dim, F = int(g["dim"]), g["fact_emb"].shape[0]
    lo, ref = _pair(g["fact_emb"], g["passage_emb"], _lo_budget(F, dim, 4))
    try:
        assert lo.fact_planes_info()["on_host"] == 2
        for k in (1, 5, 8, 16, 32):
            _assert_stage_a(lo, ref, g["q_fact"], k, f"musique1k k={k}")
        for e in (lo, ref):
            e.set_options(sim_mode=SIM_BF16)
        _assert_stage_a(lo, ref, g["q_fact"], 5, "musique1k HRAG_SIM_BF16")
    finally:
        lo.close()
        ref.close()


# ------------------------------------------------------------------------------ the bound and the fallback
def test_screen_bound_sees_every_lo_norm():
    """Unit rows, and in the last 40 rows -- inside the last 128-row step of the fill -- sign-aligned rows 4 times
    longer whose lo parts point along their queries' hi parts (the rows of test_screen_bound_follows_plane_writers, at
    its dim): against them |s4 - s1| is many times the bound E_q the other rows give, so a load that skipped that
    step's lo norms would fail the rescore's check (a counted fallback) or the byte comparison."""
    dim, F, n_long = 64, 65_536 + 100, 40
    rng = np.random.default_rng(11)
    fe = _unit(rng.standard_normal((F, dim)))
    signs = rng.choice([-1.0, 1.0], (n_long, dim))
    fe[F - n_long:] = _aligned(rng, signs, signs, scale=4.0)
    Q_long = _aligned(rng, signs, signs)                    # query j: long row j's sign pattern
    stale, fresh = _err_bound(Q_long, fe[:F - n_long]), _err_bound(Q_long, fe)
    own = np.abs(np.diagonal(_cross(Q_long, fe[F - n_long:])))
    assert np.all(own > 10 * stale) and np.all(own < fresh), (own / stale, own / fresh)
    Q_unit = _queries(fe[:F - n_long], 120, rng)
    lo, ref = _pair(fe, _unit(rng.standard_normal((4, dim))), _lo_budget(F, dim))
    try:
        for k in (1, 5, 8):
            _assert_stage_a(lo, ref, Q_long, k, f"long rows k={k}", minmax=True)
            # the long rows widen the unit queries' bands too: those may fall back, as on resident planes
            _assert_stage_a(lo, ref, Q_unit, k, f"unit queries k={k}", minmax=True, fallbacks=None)
        ids = lo.stage_a(Q_long, 1)[0]
        assert np.array_equal(ids[:, 0], F - n_long + np.arange(n_long))   # long row j is query j's best
    finally:
        lo.close()
        ref.close()


TIED_TILES = range(4, 16)      # 12 tiles that each hold 10 exact copies of one row, from row 1,024 on


def _plant_ties(fe):
    """Exact copies of row 1024 in the first 10 rows of each of TIED_TILES: a query at that row ties 120 ways at its
    best score, and its tied tiles' top-8 lists are all in the band -- more saturated tiles than a query may list, so
    its chunk falls back.  Returns the tied row."""
    v = fe[1024].copy()
    for t in TIED_TILES:
        fe[t * 256:t * 256 + 10] = v
    return v


def _tie_world(dim=64, F=65_536 + 100, seed=13):
    rng = np.random.default_rng(seed)
    fe = _unit(rng.standard_normal((F, dim)))
    return fe, _plant_ties(fe), rng


def _queries_away(fe, B, rng, first=16 * 256):
    """_queries around rows >= first only: none of them sits near the copied rows."""
    base = fe[rng.integers(first, fe.shape[0], B)]
    return _unit(base + 0.5 * rng.standard_normal(base.shape).astype(np.float32) / np.sqrt(fe.shape[1]))


@pytest.mark.parametrize("tied_chunks", [(1,), (0, 1, 2)])
def test_exact_ties_fall_back(tied_chunks):
    dim = 64
    fe, tied, rng = _tie_world(dim)
    B = 3 * 1024 - 100                                    # three 1,024-query chunks, the last ragged
    Q = _queries_away(fe, B, rng)
    for c in tied_chunks:
        Q[c * 1024 + 17] = tied
    lo, ref = _pair(fe, _unit(rng.standard_normal((4, dim))), _lo_budget(fe.shape[0], dim))
    try:
        for k in (5, 8):
            extra = _assert_stage_a(lo, ref, Q, k, f"ties in chunks {tied_chunks} k={k}",
                                    fallbacks=len(tied_chunks))
            assert extra >= len(tied_chunks) * fe.shape[0] * dim * 2   # each fallback streamed the lo plane
    finally:
        lo.close()
        ref.close()


@pytest.mark.parametrize("link_top_k", [5, 16])
def test_retrieve_resident(link_top_k):
    """retrieve_resident over three chunks (stage A of the whole call first, its fallback chunk redone) equals the
    resident handle's."""
    import torch
    from hipporag_b200 import synth
    kg = synth.make_kg(30_000, 300_000, seed=21)
    F = kg.n_facts
    assert F >= 65_536 + 400
    dim = 256
    fe = synth.unit_rows(F, dim, seed=22)
    tied = _plant_ties(fe)                                 # query 1,500 ties past the caps: its chunk falls back
    pe = synth.unit_rows(kg.n_pass, dim, seed=23)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 2100, seed=24)
    qf[1500] = tied
    lo, ref = _pair(fe, pe, _lo_budget(F, dim), kg=kg)
    try:
        dqf, dqp = torch.from_numpy(qf).cuda(), torch.from_numpy(qp).cuda()
        outs = []
        for e in (lo, ref):
            e.reset_stats()
            ids = torch.empty((qf.shape[0], 50), dtype=torch.int32, device="cuda")
            sc = torch.empty((qf.shape[0], 50), dtype=torch.float32, device="cuda")
            e.retrieve_resident(dqf, dqp, ids, sc, link_top_k=link_top_k, topk=50)
            torch.cuda.synchronize()
            outs.append((ids.cpu().numpy(), sc.cpu().numpy(), e.stats()["stage_a_fallbacks"]))
        (i0, s0, fb0), (i1, s1, fb1) = outs
        _same(i0, i1, "retrieve_resident ids")
        _same(s0, s1, "retrieve_resident scores")
        assert fb0 == fb1 and (fb0 >= 1) == (link_top_k <= 8), (fb0, fb1)
    finally:
        lo.close()
        ref.close()


# ------------------------------------------------------------------------------ rejections and the drop-in
def test_bad_placement_rejected():
    import hipporag_b200 as hb
    from hipporag_b200 import HragError, _lib
    e = hb.Engine(0)
    try:
        with pytest.raises(HragError, match="placement must be"):
            _lib.check(e._lib.hrag_set_fact_placement(e._h, 7))
    finally:
        e.close()


def test_rejections_leave_the_handle(small):
    import torch
    import hipporag_b200 as hb
    from hipporag_b200 import HragError
    kg, F, fe, pe, q = small["kg"], small["F"], small["fe"], small["pe"], small["q"]
    e = hb.Engine(0, mutable=True, fact_device_bytes=_lo_budget(F, DIM, 3), fact_lo_on_host=True)
    try:
        e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
        e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        e.load_embeddings(fe, pe)
        want = [e.stage_a(q, 5), e.stage_a(q, 16)]
        with pytest.raises(HragError, match="hrag_knn_threshold: the fact planes are held in host memory"):
            e.knn_threshold(0, q, 0.5)
        with pytest.raises(HragError, match="hrag_index_reserve: the fact planes are held in host memory"):
            e.reserve(facts=F + 10)
        with pytest.raises(HragError, match="hrag_index_append: the fact planes are held in host memory"):
            e.append(0, ent_chunk_count=kg.ent_chunk_count)
        with pytest.raises(HragError, match="hrag_index_delete: the fact planes are held in host memory"):
            e.delete(facts=[0], ent_chunk_count=kg.ent_chunk_count)
        with pytest.raises(HragError, match="pinned host memory"):
            e.export_index()
        with pytest.raises(HragError, match="pass the fp32 fact rows from host memory"):
            e.load_embeddings(torch.from_numpy(fe).cuda(), pe)
        e.set_options(sim_mode=SIM_FP32)
        with pytest.raises(HragError, match="only the tensor-core modes are available"):
            e.stage_a(q, 5)
        e.set_options(sim_mode=SIM_BF16X3)
        assert e.fact_planes_info()["on_host"] == 2
        for got, w in zip([e.stage_a(q, 5), e.stage_a(q, 16)], want):
            for g, x in zip(got, w):
                _same(g, x, "stage_a after the rejections")
    finally:
        e.close()


def test_accelerate_lo_on_host_equals_resident(golden):
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
    dim, F = int(g["dim"]), g["fact_emb"].shape[0]
    sols = []
    for lo_host in (False, True):
        rag = fake_hipporag.FakeRag(kg, g["fact_emb"], g["passage_emb"], g["q_fact"], g["q_pass"], queries)
        if lo_host:
            hipporag_b200.accelerate(rag, device=0, cache=False, fact_device_bytes=_lo_budget(F, dim, 8),
                                     fact_lo_on_host=True)
        else:
            hipporag_b200.accelerate(rag, device=0, cache=False)
        sols.append(rag.retrieve(queries, num_to_retrieve=50))
        eng = rag._b200_state["engine"]
        assert eng.fact_planes_info()["on_host"] == (2 if lo_host else 0)
        eng.close()
    for a, b in zip(*sols):
        assert a.docs == b.docs
        _same(a.doc_scores, b.doc_scores, "doc_scores")
