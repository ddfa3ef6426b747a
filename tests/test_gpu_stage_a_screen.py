"""The stage-A screen against the exact split GEMM, byte for byte.

With resident fact planes on one GPU, stage A scores every fact with the hi.hi product only, keeps the candidates that
the bound E_q on |s4 - s1| cannot rule out of the top 8 or the minimum, and rescores those with the split product at
the same query row and column.  Engine.debug_exact_stage_a runs the split GEMM over all facts on the same handle; every
case here compares the two outputs bit for bit: stage_a's ids, min-max scores and n_valid, and retrieve_resident's
passage ids and scores.  Where the screen cannot prove its candidates (caps overflowed by exact ties) the chunk falls
back to the exact path, and the stats count it.  The screen serves 65,536 facts and more (below that the split GEMM
is cheaper than the screen's extra launches), so every case here has at least that many.
"""
import numpy as np
import pytest

from tests.test_gpu_selection_exact import as_f32, exact_ints


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def _unit(x):
    x = np.asarray(x, np.float64)
    return (x / np.linalg.norm(x, axis=1, keepdims=True)).astype(np.float32)


def _engine(hb, fe, dim):
    e = hb.Engine(0)
    e.load_embeddings(fe, _unit(np.random.default_rng(5).standard_normal((4, dim))))
    return e


def _both(e, Q, k):
    """(screened, exact) stage_a outputs with the per-query (min, max) fact scores (mm_fact, B <= 1024), and the
    fallbacks the screened call counted."""
    e.reset_stats()
    got = (*e.stage_a(Q, k), e.debug_fact_minmax())
    fallbacks = e.stats()["stage_a_fallbacks"]
    e.debug_exact_stage_a(True)
    try:
        want = (*e.stage_a(Q, k), e.debug_fact_minmax())
    finally:
        e.debug_exact_stage_a(False)
    assert got[3].shape == (len(Q), 2)
    return got, want, fallbacks


def _assert_bytes(got, want, what):
    for name, g, w in zip(("ids", "scores", "n_valid", "mm_fact"), got, want):
        assert g.dtype == w.dtype and g.shape == w.shape, (what, name)
        bad = np.flatnonzero(g.view(np.uint8) != w.view(np.uint8))
        assert bad.size == 0, f"{what}: {name} differ in {bad.size} bytes"


def _queries(fe, B, rng, noise=0.5):
    """C3-shaped queries: a fact row plus Gaussian noise, normalised."""
    base = fe[rng.integers(0, fe.shape[0], B)]
    return _unit(base + noise * rng.standard_normal(base.shape).astype(np.float32) / np.sqrt(fe.shape[1]))


F_RANDOM = 65_536 + 37          # not a multiple of the 256-fact tile


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [768, 1024])
@pytest.mark.parametrize("B", [1, 1000, 1024])
def test_screen_random_unit_vectors(hb, dim, B):
    rng = np.random.default_rng(dim + B)
    fe = _unit(rng.standard_normal((F_RANDOM, dim)))
    Q = _queries(fe, B, rng)
    e = _engine(hb, fe, dim)
    try:
        for n_ctas in (0, 7, 61):
            e.debug_sim_ctas(n_ctas)
            for k in range(1, 9):
                got, want, fb = _both(e, Q, k)
                _assert_bytes(got, want, f"dim={dim} B={B} ctas={n_ctas} k={k}")
                assert fb == 0, f"random data fell back ({fb} chunks)"
    finally:
        e.close()


@pytest.mark.gpu
def test_screen_musique1k(hb, golden):
    g = golden
    pad = _unit(np.random.default_rng(10).standard_normal((F_RANDOM, int(g["dim"]))))
    e = _engine(hb, np.concatenate([g["fact_emb"], pad]), int(g["dim"]))
    try:
        for k in (1, 5, 8):
            got, want, fb = _both(e, g["q_fact"], k)
            _assert_bytes(got, want, f"musique1k k={k}")
            assert fb == 0
    finally:
        e.close()


def _bf16(x):
    """Round float32 to bfloat16, to nearest even (as __float2bfloat16_rn), kept in float32."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    u = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return u.astype(np.uint32).view(np.float32)


def _split(x):
    """The library's bf16 split x = hi + lo (k_split_bf16), in float64."""
    x = np.asarray(x, np.float32)
    hi = _bf16(x)
    return hi.astype(np.float64), _bf16(x - hi).astype(np.float64)


def _err_bound(q, f_all):
    """E_q as k_query_err computes it, per query row, for the fact rows f_all."""
    qh, ql = _split(q)
    fh, fl = _split(f_all)
    Hf, Lf = np.linalg.norm(fh, axis=1).max(), np.linalg.norm(fl, axis=1).max()
    nh, nl = np.linalg.norm(qh, axis=1), np.linalg.norm(ql, axis=1)
    steps = 5 * -(-q.shape[1] // 16)
    return (nh * Lf + nl * Hf + nl * Lf + steps * 2.0 ** -20 * (nh + nl) * (Hf + Lf)) * (1 + 2.0 ** -10)


def _cross(q, f):
    """s4 - s1 of the exact products: q_hi.f_lo + q_lo.f_hi + q_lo.f_lo, [len(q), len(f)] in float64."""
    qh, ql = _split(q)
    fh, fl = _split(f)
    return qh @ fl.T + ql @ fh.T + ql @ fl.T


def _aligned(rng, hi_signs, lo_signs, scale=1.0):
    """Rows whose stored float32 values are exactly hi + lo with hi = scale * m * hi_signs (m in [1, 2) with 8
    significant bits, above 1: exact in bf16) and lo = (7/16) ulp(hi) * lo_signs, exact in bf16 and below half an ulp, so the
    bf16 split gives back exactly this hi and lo.  Not normalised: that would make the split arbitrary again."""
    m = 1.0 + rng.integers(1, 128, hi_signs.shape) / 128.0      # hi - lo stays above 1: the same ulp
    x = scale * (m * hi_signs + (7.0 / 16.0) * 2.0 ** -7 * lo_signs)
    x = x.astype(np.float32)
    hi, lo = _split(x)
    assert np.array_equal(hi, scale * m * hi_signs) and np.array_equal(lo, scale * (7.0 / 16.0) * 2.0 ** -7 * lo_signs)
    return x


@pytest.mark.gpu
def test_screen_sign_aligned_lo_parts(hb):
    """|s4 - s1| close to E_q: each query has a cluster of 40 facts with its sign pattern, the query's lo parts
    point along its hi parts and every cluster fact's lo parts point along the query's hi parts or against them, so
    q_hi.f_lo + q_lo.f_hi comes within a few per cent of its Cauchy-Schwarz bound, with either sign of the first term:
    inside a cluster s1 is shifted against s4 by up to 0.9 E_q from fact to fact, around the 8th best and across
    tiles (some saturated).  Checked in numpy on the test's own pairs before the byte comparison."""
    dim, B, per = 768, 128, 40
    F = 65_536 + 11
    rng = np.random.default_rng(11)
    signs = rng.choice([-1.0, 1.0], (B, dim))
    rows = np.repeat(signs, per, axis=0)                              # cluster c: rows [40 c, 40 c + 40)
    rho = rng.choice([-1.0, 1.0], (B * per, 1)) * rows                # lo along or against the query's hi
    pad_signs = rng.choice([-1.0, 1.0], (F - B * per, dim))
    fe = np.concatenate([_aligned(rng, rows, rho), _aligned(rng, pad_signs, rng.choice([-1.0, 1.0], pad_signs.shape))])
    Q = _aligned(rng, signs, signs)
    E = _err_bound(Q, fe)
    cross = _cross(Q, fe[:B * per])
    ratio = np.abs(cross) / E[:, None]
    assert ratio.max() <= 1.0
    own = ratio[np.arange(B)[:, None], np.arange(B)[:, None] * per + np.arange(per)]
    assert own.max() > 0.9 and np.mean(own > 0.8) > 0.3, (own.max(), np.mean(own > 0.8))   # the lo-along half
    spread = cross[np.arange(B)[:, None], np.arange(B)[:, None] * per + np.arange(per)]
    assert np.median((spread.max(1) - spread.min(1)) / E) > 0.8           # s1 order differs from s4 order by ~E
    e = _engine(hb, fe, dim)
    try:
        for k in (1, 5, 8):
            got, want, fb = _both(e, Q, k)
            _assert_bytes(got, want, f"sign-aligned k={k}")
            assert fb == 0
        assert np.all(got[0][:, 0] // per == np.arange(B))               # each query's best is in its cluster
    finally:
        e.close()


@pytest.mark.gpu
def test_screen_near_duplicate_clusters(hb):
    """Clusters of near-duplicates (more than 8 within the band of the 8th best, inside one tile) make tiles saturated:
    every fact of such a tile is a candidate.  Clusters of 20 sit inside one tile and across a tile edge."""
    dim, F, B = 768, 256 * 256 + 100, 256
    rng = np.random.default_rng(12)
    fe = _unit(rng.standard_normal((F, dim)))
    centres = _unit(rng.standard_normal((B, dim)))
    starts = [256 * 3 + 40, 256 * 6 - 10, 256 * 11 + 3]
    for i, s in enumerate(starts):
        fe[s:s + 20] = _unit(centres[i] + 1e-4 * rng.standard_normal((20, dim)))
    Q = centres.copy()
    Q[3:] = _unit(fe[rng.integers(0, F, B - 3)] + 0.1 * rng.standard_normal((B - 3, dim)))
    e = _engine(hb, fe, dim)
    try:
        for k in (1, 4, 8):
            got, want, _ = _both(e, Q, k)
            _assert_bytes(got, want, f"clusters k={k}")
        ids = got[0]
        assert all(starts[i] <= ids[i, 0] < starts[i] + 20 for i in range(3))
    finally:
        e.close()


@pytest.mark.gpu
def test_screen_exact_ties_fall_back(hb):
    """Exact small-integer scores with 300-way ties at every level: the candidate band of the 8th best holds every
    tied fact, more than a query's cap, so each chunk falls back to the exact path, counted in the stats, and the
    outputs are still those of the exact path."""
    dim, M, B = 40, 65_536 + 100, 130
    rng = np.random.default_rng(13)
    Qi = exact_ints(rng, (B, dim))
    Qi[Qi == 0] = 1
    Ei = exact_ints(rng, (M, dim))
    block = 300
    for r in range(0, M, block):                          # 300 copies of each query 0 best-row level
        Ei[r:r + block] = np.sign(Qi[0]) * (3 - (r // block) % 3)
    fe, Q = as_f32(Ei), as_f32(Qi)
    e = _engine(hb, fe, dim)
    try:
        # stage_a runs B = 130 queries as one chunk
        got, want, fb = _both(e, Q, 8)
        _assert_bytes(got, want, "exact ties")
        assert fb == 1, fb
    finally:
        e.close()


@pytest.mark.gpu
def test_screen_retrieve_resident(hb):
    """retrieve_resident (two 1,024-query chunks and a ragged third, overlapped) gives the same passage ids and scores
    with the screen as with the exact stage A."""
    import torch
    from hipporag_b200 import synth
    kg = synth.make_kg(30_000, 300_000, seed=21)
    assert kg.n_facts >= 65_536
    dim = 768
    fe = synth.unit_rows(kg.n_facts, dim, seed=22)
    pe = synth.unit_rows(kg.n_pass, dim, seed=23)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 2100, seed=24)
    e = hb.Engine(0)
    try:
        e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
        e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        e.load_embeddings(fe, pe)
        dev = torch.device("cuda", 0)
        dqf, dqp = torch.from_numpy(qf).to(dev), torch.from_numpy(qp).to(dev)
        outs = []
        for exact in (False, True):
            e.debug_exact_stage_a(exact)
            e.reset_stats()
            ids = torch.empty((qf.shape[0], 50), dtype=torch.int32, device=dev)
            sc = torch.empty((qf.shape[0], 50), dtype=torch.float32, device=dev)
            e.retrieve_resident(dqf, dqp, ids, sc, link_top_k=5, topk=50)
            torch.cuda.synchronize()
            outs.append((ids.cpu().numpy(), sc.cpu().numpy(), e.stats()["stage_a_fallbacks"]))
        e.debug_exact_stage_a(False)
        (i0, s0, fb), (i1, s1, _) = outs
        assert fb == 0
        assert np.array_equal(i0, i1)
        assert np.array_equal(s0.view(np.uint32), s1.view(np.uint32))
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["whole", "streamed"])
def test_screen_bound_follows_plane_writers(hb, layout):
    """The screen's bound rests on the largest fact-plane row norms, which every writer keeps: a whole or streamed
    load of unit rows, then an in-place append of rows 4 times longer whose lo parts point along their queries' hi
    parts.  Against those rows |s4 - s1| is many times the bound the loaded rows alone would give, so a writer that
    left the norm maxima stale would fail the rescore's check (a counted fallback) or the byte comparison."""
    from tests.test_gpu_index_update import _append, _base, _batch, _engine_layout
    ix = _base(n_nodes=30_000, n_edges=300_000)
    assert ix.fe.shape[0] >= 65_536
    dim = ix.fe.shape[1]
    e = _engine_layout(ix, layout)
    try:
        rng = np.random.default_rng(14)
        Q = _unit(ix.fe[rng.integers(0, ix.fe.shape[0], 200)] + 0.3 * rng.standard_normal((200, dim)))
        got, want, fb = _both(e, Q, 8)
        _assert_bytes(got, want, f"{layout} load")
        assert fb == 0
        bt = _batch(ix, rng)
        signs = rng.choice([-1.0, 1.0], bt.fe.shape)
        bt.fe[:] = _aligned(rng, signs, signs, scale=4.0)
        Q2 = _aligned(rng, signs, signs)                            # query j: appended fact j's sign pattern
        stale, fresh = _err_bound(Q2, ix.fe), _err_bound(Q2, np.concatenate([ix.fe, bt.fe]))
        own = np.abs(np.diagonal(_cross(Q2, bt.fe)))
        assert np.all(own > 10 * stale) and np.all(own < fresh), (own / stale, own / fresh)
        _append(e, bt)
        got, want, fb = _both(e, Q2, 8)
        _assert_bytes(got, want, f"{layout} load + append")
        assert fb == 0
        assert np.array_equal(got[0][:, 0], ix.fe.shape[0] + np.arange(len(Q2)))   # appended fact j is query j's best
    finally:
        e.close()
