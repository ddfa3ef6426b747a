"""Selection kernels on exact scores: every top-k, min-max and threshold kernel against a float32 oracle, bit for bit.

Embeddings and queries are small integers / 4 (entries in {-3, ..., 3} / 4).  Every product is then a multiple of
1/16, every partial sum of a dot product up to d = 1024 fits in 14 significant bits, and bf16 holds every entry, so
the bf16 split is hi = x, lo = 0.  Every similarity mode (SIM_FP32, SIM_BF16X3, SIM_BF16) must therefore return the
integer dot product / 16 exactly, whatever its accumulation order, and min-max normalisation is reproduced bit for bit
by numpy in float32 ((s - min) / (max - min), correctly rounded like __fdiv_rn).  Ties are exact and are planted where
kernels go wrong: across the four lanes of a wgmma quad, across 256-column tile edges, more than 8 inside one tile,
at the top-k / threshold cut, and in the padding of a ragged last tile.  All assertions on ids and scores are
equalities; only the seed-selection test (which runs a PPR solve) uses the near-tie tolerant checker.
"""
import numpy as np
import pytest

from oracle import ppr, retrieve
from tests.util import assert_topk_matches

SMALL_K = tuple(range(1, 9))          # selected in the GEMM epilogue / k_row_minmax_topk
RADIX_K = (9, 16, 31, 32)             # k_row_topk + k_topk_normalize


# ------------------------------------------------------------------------------ host-side oracle
def exact_ints(rng, shape, lo=-3, hi=3):
    return rng.integers(lo, hi + 1, size=shape, dtype=np.int64)


def as_f32(a):
    """Integer matrix -> the float32 vectors the engine sees (exact: entries are multiples of 1/4)."""
    return np.ascontiguousarray(np.asarray(a, dtype=np.float32) / np.float32(4))


def raw_scores(Qi, Ei):
    """[B, M] float32 dot products of as_f32(Qi) and as_f32(Ei), from an int64 matmul scaled once."""
    return ((np.asarray(Qi, np.int64) @ np.asarray(Ei, np.int64).T).astype(np.float32) / np.float32(16))


def minmax32(raw):
    """misc_utils.min_max_normalize per row, in float32 (the reference's dtype): all-equal rows -> 1."""
    raw = np.asarray(raw, np.float32)
    mn = raw.min(axis=1, keepdims=True)
    rg = raw.max(axis=1, keepdims=True) - mn
    with np.errstate(invalid="ignore", divide="ignore"):
        out = (raw - mn) / rg
    out[np.broadcast_to(rg == 0, out.shape)] = np.float32(1)
    return out.astype(np.float32)


def ranking(s):
    """Per row: score descending, then index ascending (the library's documented tie policy)."""
    return np.argsort(-np.asarray(s), axis=-1, kind="stable")


def expected_topk(s, order, k):
    """(ids, scores, n_valid) of a [B, k] top-k output: -1 / 0.0 past the M real entries."""
    B, M = s.shape
    kk = min(k, M)
    ids = np.full((B, k), -1, np.int32)
    sc = np.zeros((B, k), np.float32)
    ids[:, :kk] = order[:, :kk]
    sc[:, :kk] = np.take_along_axis(s, order[:, :kk].astype(np.int64), axis=1)
    return ids, sc, np.full(B, kk, np.int32)


def assert_same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    if not np.array_equal(got, want):
        bad = np.nonzero((got != want).reshape(got.shape[0], -1).any(axis=1))[0] if got.ndim else [0]
        r = int(bad[0])
        col = np.nonzero(np.atleast_1d(got[r] != want[r]))[0]
        c = int(col[0]) if col.size else 0
        raise AssertionError(f"{what}: {len(bad)} rows differ; row {r} from column {c}: got "
                             f"{np.atleast_1d(got[r])[c:c + 8]}, want {np.atleast_1d(want[r])[c:c + 8]}")


# ------------------------------------------------------------------------------ CPU: the premise itself
def test_exact_premise_on_host():
    rng = np.random.default_rng(0)
    for dim in (8, 40, 136, 768, 1024):
        Ei = exact_ints(rng, (300, dim))
        Qi = exact_ints(rng, (5, dim))
        Ei[7] = 3                                        # the largest possible dot products: 9 * dim / 16
        Qi[0] = 3
        Qi[1] = -3
        got = as_f32(Qi) @ as_f32(Ei).T                  # float32 BLAS, any summation order
        want = raw_scores(Qi, Ei)
        assert got.dtype == np.float32 and np.array_equal(got, want), dim
        assert want[0, 7] == 9 * dim / 16 and want[1, 7] == -9 * dim / 16
        assert np.array_equal((Qi @ Ei.T).astype(np.float64) / 16, want.astype(np.float64))
        # bf16 (the top 16 bits of a float32) holds every entry: the split leaves lo = 0
        bits = as_f32(Ei).view(np.uint32)
        assert np.all(bits & 0xffff == 0)
    # min-max in float32 is correctly rounded and maps distinct scores to distinct values
    n = minmax32(np.array([[-1.5, 0.25, 0.0, 2.0, -1.5]], np.float32))
    assert n.dtype == np.float32 and n[0, 0] == 0 and n[0, 3] == 1 and n[0, 4] == 0
    assert n[0, 1] == np.float32(1.75) / np.float32(3.5)
    assert np.all(minmax32(np.zeros((2, 3), np.float32)) == 1)
    # ranking: score descending, then index ascending; -0.0 ties with +0.0
    s = np.array([[0.5, 1.0, 0.5, 1.0, -0.0, 0.0, -2.0, 0.0]], np.float32)
    assert ranking(s)[0].tolist() == [1, 3, 0, 2, 4, 5, 7, 6]
    ids, sc, nv = expected_topk(s, ranking(s), 10)
    assert ids[0].tolist() == [1, 3, 0, 2, 4, 5, 7, 6, -1, -1] and sc[0, 8:].tolist() == [0, 0] and nv[0] == 8


# ------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def _fact_engine(hb, Ei):
    e = hb.Engine(0)
    e.load_embeddings(as_f32(Ei), as_f32(np.ones((4, Ei.shape[1]), np.int64)))
    return e


def _routes(hb, dim):
    """(name, sim_mode, keep_scores) of every stage-A route an engine of this dim can take."""
    if dim % 8:
        return [("k_sim_fp32 (dim % 8 != 0)", hb.SIM_BF16X3, False)]
    return [("fused bf16x3", hb.SIM_BF16X3, False), ("fused bf16", hb.SIM_BF16, False),
            ("materialised bf16x3", hb.SIM_BF16X3, True), ("materialised bf16", hb.SIM_BF16, True),
            ("fp32", hb.SIM_FP32, False)]


def check_stage_a_routes(hb, e, Qi, Ei, what, ks=SMALL_K + RADIX_K):
    """Every route, every k: ids, min-max scores and n_valid equal the float32 oracle; the materialised score matrix
    of the last chunk equals the integer dot products / 16."""
    Q = as_f32(Qi)
    raw = raw_scores(Qi, Ei)
    norm = minmax32(raw)
    order = ranking(raw)
    try:
        for name, mode, keep in _routes(hb, Ei.shape[1]):
            e.set_options(sim_mode=mode)
            e.debug_keep_scores(keep)
            for k in ks:
                idx, sc, nv = e.stage_a(Q, k)
                want_idx, want_sc, want_nv = expected_topk(norm, order, k)
                tag = f"{what}, {name}, k={k}"
                assert_same(nv, want_nv, tag + ": n_valid")
                assert_same(idx, want_idx, tag + ": ids")
                assert_same(sc, want_sc, tag + ": scores")
            if keep or max(ks) > 8 or mode == hb.SIM_FP32 or Ei.shape[1] % 8:
                got = e.debug_scores(0)                 # rows of the last chunk
                assert got.shape[0] > 0
                assert_same(got, raw[raw.shape[0] - got.shape[0]:], f"{what}, {name}: raw scores")
    finally:
        e.debug_keep_scores(False)
        e.set_options(sim_mode=hb.SIM_BF16X3)


def _top_row(q):
    """The row with the largest possible dot product with q: 3 * sign(q)."""
    return 3 * np.sign(q)


# (M facts, dim, B queries): every M class around the 256-column tile and the 8-best register list, every dim class
# (one ragged k-block, k-blocks ragged against the 32- and 64-column stages), query counts around the 128-query tile,
# dims that are not a multiple of 8 (k_sim_fp32 whatever the mode) and one batch across the 1024-query chunk
STAGE_A_CASES = [
    (1, 8, 129), (2, 24, 128), (7, 40, 127), (8, 136, 1), (9, 768, 129),
    (255, 8, 127), (256, 24, 129), (257, 40, 128), (511, 136, 129), (513, 768, 127),
    (1003, 8, 128), (1003, 24, 1), (1003, 40, 129), (1003, 136, 127), (1003, 768, 128),
    (257, 12, 129), (1003, 100, 128), (1003, 40, 1025),
]


@pytest.mark.gpu
@pytest.mark.parametrize("M,dim,B", STAGE_A_CASES)
def test_stage_a_routes_agree_exactly(hb, M, dim, B):
    rng = np.random.default_rng(M * 7919 + dim * 31 + B)
    Ei = exact_ints(rng, (M, dim))
    Qi = exact_ints(rng, (B, dim))
    Qi[0][Qi[0] == 0] = 1
    # query 0: its best row duplicated across the lanes of one quad (columns 1, 2, 5, 6 hold lanes 0..3),
    # across tile edges and into the ragged last tile
    dup = [c for c in (0, 1, 2, 5, 6, 255, 256, 511, 512, 767, 768, M - 1) if c < M]
    Ei[dup] = _top_row(Qi[0])
    if B > 1 and M > 311:
        # query 1: its best row 12 times inside tile 1 -- the top-8 cut falls inside the tie
        Qi[1][Qi[1] == 0] = -1
        Ei[300:312] = _top_row(Qi[1])
    if B > 2:
        Qi[B - 1] = 0                                    # range 0: every score 1.0, ids 0..k-1
    if B > 128:
        Qi[128] = Qi[0]                                  # the same planted ties in the second query tile
    raw = raw_scores(Qi, Ei)
    assert np.all(raw[0, dup] == raw[0].max())
    if B > 1 and M > 311:
        assert np.count_nonzero(raw[1] == raw[1].max()) >= 12
    e = _fact_engine(hb, Ei)
    check_stage_a_routes(hb, e, Qi, Ei, f"M={M} dim={dim} B={B}")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [8, 40, 136, 100])
@pytest.mark.parametrize("M", [1, 7, 257, 513, 1003])
def test_stage_a_sign_edges(hb, dim, M):
    """All-positive and all-negative rows of a ragged last tile: a padded column's 0.0 would become the min or the
    max.  All-equal rows and the zero query: range 0, scores 1.0, ids 0..k-1."""
    rng = np.random.default_rng(M + dim)
    Ei = exact_ints(rng, (M, dim), 1, 3)                 # every entry > 0
    Qi = np.stack([exact_ints(rng, dim, 1, 3), -exact_ints(rng, dim, 1, 3), np.zeros(dim, np.int64),
                   exact_ints(rng, dim)])
    raw = raw_scores(Qi, Ei)
    assert raw[0].min() > 0 and raw[1].max() < 0 and np.all(raw[2] == 0)
    e = _fact_engine(hb, Ei)
    check_stage_a_routes(hb, e, Qi, Ei, f"positive rows M={M} dim={dim}")
    e.close()
    e = _fact_engine(hb, -Ei)                             # every entry < 0: the signs of rows 0 and 1 swap
    check_stage_a_routes(hb, e, Qi, -Ei, f"negative rows M={M} dim={dim}")
    e.close()
    same = np.repeat(exact_ints(rng, (1, dim)), M, axis=0)
    e = _fact_engine(hb, same)
    check_stage_a_routes(hb, e, Qi, same, f"all-equal rows M={M} dim={dim}")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [8, 40, 768])
def test_stage_a_zero_block_at_cut(hb, dim):
    """Three positive scores, then 40 scores of exactly 0.0, the rest negative: the top-k cut for every k in 4..32
    falls inside the zero block, which must be ordered by index.  Half of the zeros are sums of negative zeros only
    (-0.0 in IEEE arithmetic), half come from cancellation (+0.0); float_to_ordered must not separate them."""
    M, h = 1003, dim // 2
    rng = np.random.default_rng(dim)
    Qi = np.zeros((3, dim), np.int64)
    Qi[0, :h] = -exact_ints(rng, h, 1, 3)                # negative on the first half, 0 on the second
    Qi[1, :h] = -1
    Ei = np.zeros((M, dim), np.int64)
    Ei[:, :h] = exact_ints(rng, (M, h), 1, 3)            # default: every score < 0
    Ei[:, h:] = exact_ints(rng, (M, dim - h))
    pos = [40, 700, 1002]
    Ei[pos, :h] = -exact_ints(rng, (3, h), 1, 3)
    zeros = [1, 2, 5, 6, 9, 13, 100, 254, 255, 256, 257, 300, 301, 302, 303, 304, 305, 306, 307, 400, 510, 511, 512,
             513, 600, 601, 766, 767, 768, 769, 800, 801, 900, 901, 990, 997, 998, 999, 1000, 1001]
    for j, c in enumerate(zeros):
        if j % 2 == 0:                                   # 0 on the query's support, negative elsewhere: -0 * x, 0 * -x
            Ei[c, :h] = 0
            Ei[c, h:] = -exact_ints(rng, dim - h, 1, 3)
        else:                                            # q0 * (-q1) + q1 * q0 = 0 on the support
            Ei[c, :h] = 0
            Ei[c, 0], Ei[c, 1] = -Qi[0, 1], Qi[0, 0]
    raw = raw_scores(Qi, Ei)
    assert np.count_nonzero(raw[0] > 0) == 3 and np.count_nonzero(raw[0] == 0) == len(zeros)
    assert np.all(raw[2] == 0)
    e = _fact_engine(hb, Ei)
    check_stage_a_routes(hb, e, Qi, Ei, f"zero block dim={dim}")
    e.close()


# ------------------------------------------------------------------------------ k_row_topk at every size class
def _level_rows(rng, M, dim, block=300):
    """Rows whose score against the query (3, 1, 0, ...) is 3a + b for their first two entries (a, b): the best 300 rows share
    the top level, the next 300 the next one, and so on, at random indices -- every k below is inside a 300-way tie."""
    levels = np.repeat(np.arange(12, -13, -1), block)[:M]
    a = np.empty(M, np.int64)
    for lv in np.unique(levels):
        cand = [x for x in range(-3, 4) if -3 <= lv - 3 * x <= 3]
        a[levels == lv] = rng.choice(cand, size=int(np.count_nonzero(levels == lv)))
    E = exact_ints(rng, (M, dim))
    E[:, 0], E[:, 1] = a, levels - 3 * a
    return E[rng.permutation(M)]


TOPK_K = (1, 7, 8, 9, 255, 256, 257, 1023, 1024, 1025, 2047, 2048)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 5, 2048, 2049, 5000])
def test_topk_similarity_every_size_class(hb, M):
    dim = 8
    rng = np.random.default_rng(M)
    Ei = _level_rows(rng, M, dim)
    level_query = np.array([3, 1, 0, 0, 0, 0, 0, 0])
    Qi = np.stack([level_query, exact_ints(rng, dim), np.zeros(dim, np.int64), -level_query])
    raw = raw_scores(Qi, Ei)
    order = ranking(raw)
    for k in TOPK_K:
        if k < M:
            assert raw[0, order[0, k - 1]] == raw[0, order[0, k]], k      # the cut is inside a tie
    e = _fact_engine(hb, Ei)
    for mode in (hb.SIM_BF16X3, hb.SIM_FP32):
        e.set_options(sim_mode=mode)
        for k in TOPK_K:
            ids, sc = e.topk_similarity(0, as_f32(Qi), k)
            want_ids, want_sc, _ = expected_topk(raw, order, k)
            assert_same(ids, want_ids, f"M={M} mode={mode} k={k}: ids")
            assert_same(sc, want_sc, f"M={M} mode={mode} k={k}: raw scores")
    e.close()


# ------------------------------------------------------------------------------ threshold epilogue
def _threshold_case():
    """1025 queries (two 1024-query chunks) x 1003 rows, d = 40, threshold 2.5 = 40 / 16.  Queries 0 and 700 each
    clear it on more than 512 rows (600 rows carry 3 on the eight coordinates where those queries are 3)."""
    rng = np.random.default_rng(77)
    M, dim, B = 1003, 40, 1025
    Ei = exact_ints(rng, (M, dim))
    over_rows = rng.choice(M, 600, replace=False)
    Ei[over_rows, :8] = 3
    Qi = exact_ints(rng, (B, dim))
    for q in (0, 700):
        Qi[q] = 0
        Qi[q, :8] = 3
    Qi[1024, :8] = -np.abs(Qi[1024, :8])             # the second chunk's only query stays below the cap
    return Ei, Qi, np.float32(2.5)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16x3", "bf16"])
def test_knn_threshold_exact(hb, mode):
    Ei, Qi, thr = _threshold_case()
    raw = raw_scores(Qi, Ei)
    order = ranking(raw)
    count = (raw >= thr).sum(axis=1)
    over = count > 512
    assert np.nonzero(over)[0].tolist()[:2] == [0, 700] and over.sum() < 20
    assert 0 < count[1024] <= 512 and count[1024] + count[0] > 512
    assert np.count_nonzero((raw == thr).any(axis=1)) > 100         # scores exactly at the threshold
    e = _fact_engine(hb, Ei)
    e.set_options(sim_mode=hb.SIM_BF16X3 if mode == "bf16x3" else hb.SIM_BF16)
    ties_at_cut = 0
    for kmax in (16, 512):
        ids, sc, found = e.knn_threshold(0, as_f32(Qi), float(thr), kmax)
        assert_same(found, count.astype(np.int32), f"{mode} kmax={kmax}: n_found")
        want_ids, want_sc, _ = expected_topk(raw, order, kmax)
        n = np.minimum(count, kmax)
        keep = np.arange(kmax)[None, :] < n[:, None]
        want_ids = np.where(keep, want_ids, -1)
        want_sc = np.where(keep, want_sc, np.float32(0))
        assert_same(ids[~over], want_ids[~over], f"{mode} kmax={kmax}: ids")
        assert_same(sc[~over], want_sc[~over], f"{mode} kmax={kmax}: scores")
        # an overflowing query returns the best of the 512 candidates its buffer kept, in rank order
        for q in np.nonzero(over)[0]:
            got = ids[q][ids[q] >= 0]
            assert got.size == kmax and np.unique(got).size == kmax
            assert np.all(raw[q, got] >= thr) and np.array_equal(sc[q, :kmax], raw[q, got])
            assert got.tolist() == sorted(got.tolist(), key=lambda j: (-raw[q, j], j))
        if kmax == 16:
            cut = (count > kmax) & ~over
            ties_at_cut = np.count_nonzero(cut & (raw[np.arange(len(raw)), order[:, kmax - 1]]
                                                 == raw[np.arange(len(raw)), order[:, kmax]]))
    assert ties_at_cut > 10
    e.close()


@pytest.mark.gpu
def test_retrieve_knn_min_score_overflow_redo(hb):
    """retrieve_knn(min_score=...) end to end.  Keys and queries are +-1 in d = 64, so the unit rows are +-1/8 and
    every cosine is an exact multiple of 1/64.  Query 7 clears the threshold on more than 512 keys: its list must come
    back through the exact redo path, equal to the first min(k, 128) keys >= the threshold."""
    from hipporag_b200.knn import retrieve_knn
    rng = np.random.default_rng(5)
    M, dim, B = 1003, 64, 50
    keys = rng.choice([-1, 1], size=(M, dim)).astype(np.int64)
    qs = rng.choice([-1, 1], size=(B, dim)).astype(np.int64)
    keys[rng.choice(M, 600, replace=False), :48] = qs[7, :48]
    keys[11] = keys[3]                                   # duplicate keys: lower index first
    qs[20] = keys[3]
    thr = 16 / 64
    raw = (qs @ keys.T).astype(np.float32) / np.float32(64)
    order = ranking(raw)
    count = (raw >= thr).sum(axis=1)
    assert count[7] > 512 and count.min() > 0
    key_ids = [f"k{i}" for i in range(M)]
    e = hb.Engine(0)
    redo = []
    topk_similarity = e.topk_similarity

    def spy(which, q, k):
        redo.append(q.shape[0])
        return topk_similarity(which, q, k)

    e.topk_similarity = spy
    for k in (2047, 50):
        redo.clear()
        res = retrieve_knn([f"q{i}" for i in range(B)], key_ids, qs.astype(np.float32), keys.astype(np.float32),
                           k=k, engine=e, min_score=thr)
        assert redo == [int((count > 512).sum())]        # the overflow redo ran, once, for every overflowing query
        for i in range(B):
            n = int(min(count[i], k, 128))
            ids, sc = res[f"q{i}"]
            assert ids == [f"k{j}" for j in order[i, :n]], (k, i)
            assert np.array_equal(np.array(sc, np.float32), raw[i, order[i, :n]]), (k, i)
    assert res["q20"][0][:2] == ["k3", "k11"]
    e.close()


# ------------------------------------------------------------------------------ the three DPR min-max copies
@pytest.mark.gpu
@pytest.mark.parametrize("n_nodes", [20_470, 20_490])          # P = 2047, 2049 passages
def test_dpr_minmax_copies_agree(hb, n_nodes):
    """A DPR row is min-maxed by k_minmax_apply (stage B with no kept facts), by the fp32-solver gather (<= 16
    queries) and by the mixed-solver gather (> 16 queries): all three must equal the float32 oracle bit for bit."""
    from hipporag_b200 import synth
    kg = synth.make_kg(n_nodes, 6 * n_nodes, seed=11)
    P, dim = kg.n_pass, 8
    rng = np.random.default_rng(n_nodes)
    Ep = exact_ints(rng, (P, dim))
    Ep[P - 3:] = Ep[[0, 1023, 1024]]                      # duplicated passages on both sides of every cut
    Ef = exact_ints(rng, (kg.n_facts, dim))
    Qp = exact_ints(rng, (40, dim))
    Qp[3] = 0                                            # range 0: every passage scores 1.0
    Qf = exact_ints(rng, (40, dim))
    e = hb.Engine(0)
    e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    e.load_embeddings(as_f32(Ef), as_f32(Ep))
    raw_p = raw_scores(Qp, Ep)
    norm_p = minmax32(raw_p)
    order_p = ranking(raw_p)
    assert_same(e.similarity(1, as_f32(Qp)), norm_p, "hrag_similarity(passages)")
    assert_same(e.similarity(0, as_f32(Qf)), minmax32(raw_scores(Qf, Ef)), "hrag_similarity(facts)")
    kept, kscore, _ = e.stage_a(as_f32(Qf), 5)
    kept[4] = -1                                         # the filter kept nothing: DPR fallback
    flags = np.zeros(40, np.uint8)
    flags[[1, 3, 17, 33, 39]] = 1
    dpr5, dpr40 = [1, 3, 4], [1, 3, 4, 17, 33, 39]
    for topk in [t for t in (1, P - 1, P, P + 1, 2048) if t <= 2048]:
        want_ids, want_sc, _ = expected_topk(norm_p, order_p, topk)
        ids_a, sc_a = e.stage_b(as_f32(Qp), np.zeros((40, 0), np.int32), np.zeros((40, 0), np.float32), topk=topk)
        assert_same(ids_a, want_ids, f"P={P} topk={topk} k_minmax_apply: ids")
        assert_same(sc_a, want_sc, f"P={P} topk={topk} k_minmax_apply: scores")
        e.reset_stats()
        ids_b, sc_b = e.stage_b(as_f32(Qp[:5]), kept[:5], kscore[:5], flags[:5], topk=topk)
        st = e.stats()
        assert st["ppr_columns"] < 32 * st["ppr_sweeps"]                # the fp32 solver
        assert_same(ids_b[dpr5], want_ids[dpr5], f"P={P} topk={topk} fp32-solver gather: ids")
        assert_same(sc_b[dpr5], want_sc[dpr5], f"P={P} topk={topk} fp32-solver gather: scores")
        e.reset_stats()
        ids_c, sc_c = e.stage_b(as_f32(Qp), kept, kscore, flags, topk=topk)
        st = e.stats()
        assert st["ppr_columns"] == 32 * st["ppr_sweeps"]               # the mixed solver
        assert_same(ids_c[dpr40], want_ids[dpr40], f"P={P} topk={topk} mixed-solver gather: ids")
        assert_same(sc_c[dpr40], want_sc[dpr40], f"P={P} topk={topk} mixed-solver gather: scores")
    e.close()


# ------------------------------------------------------------------------------ seed selection at the link_top_k cut
@pytest.mark.gpu
def test_seed_selection_tie_at_link_top_k(hb):
    """Phrase weights that tie exactly on the link_top_k cut: k_seed_entities must keep the lower vertex ids
    (weight desc, vertex id asc).  Keeping another phrase of the tie moves the PPR ranking far past the near-tie
    allowance, which the test checks on the oracle itself."""
    from hipporag_b200 import synth
    kg = synth.make_kg(2000, 20_000, seed=5)
    n, dim = kg.n_nodes, 16
    rng = np.random.default_rng(3)
    F = 40
    # fact scores against q = (4, 1, 0, ...) are 4a + b for fact row (a, b, ...): A 15, B 13, C = D 12, E 11, the
    # others <= 7, fact 0 at -15 (so normalised = (s + 15) / 30)
    A, B_, C_, D_, E_ = 10, 3, 20, 25, 7
    Ef = exact_ints(rng, (F, dim))
    Ef[:, 0] = rng.integers(-3, 2, F)
    Ef[0, :2] = (-3, -3)
    for f, (a, b) in ((A, (3, 3)), (B_, (3, 1)), (C_, (3, 0)), (D_, (3, 0)), (E_, (3, -1))):
        Ef[f, :2] = (a, b)
    q_fact = np.zeros(dim, np.int64)
    q_fact[:2] = (4, 1)
    live = rng.choice(np.arange(1000, 1700), size=(F, 2), replace=False)
    subj, obj = live[:, 0].astype(np.int32), live[:, 1].astype(np.int32)
    a1, b1, tx, shared, ty, tz, e1, e2 = 100, 150, 200, 900, 300, 600, 400, 450
    for f, s, o in ((A, a1, a1), (B_, b1, tx), (C_, shared, ty), (D_, shared, tz), (E_, e1, e2)):
        subj[f], obj[f] = s, o                            # fact A: subject == object
    cc = kg.ent_chunk_count.copy()
    for v, c in ((a1, 1), (b1, 1), (tx, 2), (shared, 2), (ty, 2), (tz, 2), (e1, 2), (e2, 1)):
        cc[v] = c                                        # powers of two: fp32 and float64 division agree
    # weights: a1 1, b1 28/30, e2 26/30, tx 28/60, {ty 300, tz 600, shared 900} 27/60, e1 26/60
    Ep = exact_ints(rng, (kg.n_pass, dim))
    Qp = exact_ints(rng, (2, dim))
    e = hb.Engine(0)
    e.load_graph(n, kg.edge_src, kg.edge_dst, kg.edge_w)
    e.load_tables(kg.passage_vid, subj, obj, cc)
    e.load_embeddings(as_f32(Ef), as_f32(Ep))
    Qf = as_f32(np.stack([q_fact, q_fact]))
    idx, score, _ = e.stage_a(Qf, 5)
    assert idx[0].tolist() == [A, B_, C_, D_, E_] and score[0, 2] == score[0, 3]
    Pm = ppr.transition_matrix(ppr.symmetric_weights(n, kg.edge_src, kg.edge_dst, kg.edge_w))[0]
    tables = retrieve.Tables(n, kg.passage_vid, subj, obj, cc)
    fs = retrieve.fact_scores(as_f32(Ef), Qf[0])
    topk = 50
    holes = np.full_like(idx, -1)
    holes[:, 1:4] = idx[:, 1:4]                          # kept-index lists with -1 holes: B, C, D
    hole_score = np.where(holes >= 0, score, np.float32(0.99))
    for kept_idx, kept_score, ltk, want_seeds, other in (
            (idx, score, 5, {a1, b1, e2, tx, ty}, (ty, shared)),
            (holes, hole_score, 4, {b1, tx, ty, tz}, (ty, shared))):
        ids, scores = e.stage_b(as_f32(Qp), kept_idx, kept_score, link_top_k=ltk, topk=topk)
        kept = [int(f) for f in kept_idx[0] if f >= 0]
        for q in range(2):
            ps = retrieve.passage_scores(as_f32(Ep), as_f32(Qp[q]))
            r, seeds = retrieve.seed_vector(tables, fs, kept, ps, ltk, 0.05)
            assert set(seeds) == want_seeds
            pi = ppr.ppr_power(Pm, r, 0.5)[kg.passage_vid]
            assert_topk_matches(ids[q], scores[q], pi, topk, what=f"link_top_k={ltk} query {q}")
            # the same weight on the highest vertex id of the tie instead: a different answer
            r_alt = r.copy()
            r_alt[other[1]], r_alt[other[0]] = r[other[0]], 0.0
            pi_alt = ppr.ppr_power(Pm, r_alt, 0.5)[kg.passage_vid]
            alt = retrieve.order_desc(pi_alt, topk)
            with pytest.raises(AssertionError):
                assert_topk_matches(alt, pi_alt[alt], pi, topk)
    e.close()
