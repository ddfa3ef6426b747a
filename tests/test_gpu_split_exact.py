"""The split-bf16 similarity GEMM (K2, k_sim_tc) against exact references whose lo planes are not zero.

K2 stores each vector as x = hi + lo (both bf16).  SIM_BF16X3 accumulates the four products q_lo.e_lo, q_hi.e_lo,
q_lo.e_hi and q_hi.e_hi per k-block; SIM_BF16 accumulates q_hi.e_hi only.  The inputs here are built so that every
stored float32 splits into a known hi and lo, and every partial sum of every dot product is exact in fp32.  Both modes
must then return the float64 value of their own products bit for bit, on every route that runs the GEMM.  Three
families of inputs:

  A  fact lo only: fact entries a/4 + c 2^-12 (a in {+-1, +-2, +-3}, c in -3..3, |c| <= 1 where |a| = 1, since the bf16
     grid is finer below 0.25), queries in {-2..2}/4 (q_lo = 0).  Exercises q_hi.e_lo.
  B  query lo only: the mirror image.  Exercises q_lo.e_hi.
  C  a lo.lo witness: hi = +-1, lo = +-2^-10.  The queries are non-zero on two columns of each 16-column group, where
     the facts' hi parts cancel q_hi.e_hi, so every score is the cross terms plus the lo.lo sum, with no large
     accumulator.  Only this family changes its answer when lo.lo is dropped.

Random data of these kinds ranks the same under both modes, so rows whose hi parts are identical and whose lo parts
differ are planted for query 0 (and its copy in the second 128-query tile): inside one wgmma quad, across 256-column
tile edges, at the top-k cut, at the minimum and at the knn_threshold threshold.

The CPU tests check these premises, and for each plausible defect of the mainloop (a product dropped, an operand read
from the wrong plane, a lo k-offset or row off by one step, the lo part of a ragged last k-block read as zero) that
the numpy output the GPU tests compare against would change.

The last part measures the accumulation model under the stage-A screen's bound E_q (DESIGN.md section 4, K2) on the
hardware: the materialised SIM_BF16 / SIM_BF16X3 scores come from the same mainloops as the screen's s1 and s4.
"""
import numpy as np
import pytest

from tests.test_gpu_selection_exact import assert_same, expected_topk, minmax32, ranking
from tests.test_gpu_stage_a_screen import _aligned, _bf16, _split, _unit

SMALL_K = tuple(range(1, 9))          # the GEMM's fused top-8 epilogue (FUSE 1)
RADIX_K = (9, 16, 31, 32)             # materialised scores + k_row_topk
LO_A = 2.0 ** -12                     # the lo unit of families A and B
LO_C = 2.0 ** -10                     # the lo part of family C
ACC_STEP = 2.0 ** -20                 # k_query_err's relative accumulation error per k16 wgmma step


# ------------------------------------------------------------------------------ the three families
def _lo_units(rng, a):
    """c in -3..3, or -1..1 where |a| = 1: a/4 + c 2^-12 then rounds to a/4 in bf16 (c 2^-12 < half its ulp)."""
    c = rng.integers(-3, 4, a.shape)
    one = np.abs(a) == 1
    c[one] = rng.integers(-1, 2, int(one.sum()))
    return c


def _nonzero_a(rng, shape):
    return rng.choice(np.array([-3, -2, -1, 1, 2, 3]), shape)


def _sign(x):
    return np.where(np.asarray(x) >= 0, 1, -1)


def _planted_cols(M):
    """Columns of query 0's planted best rows -- lanes 0..3 of one quad (columns 1, 2, 5, 6), both sides of every tile
    edge, the ragged last tile, and twelve more in tile 1, so that the top-8 cut falls inside them -- and of its
    planted worst rows."""
    top = [c for c in (1, 2, 5, 6, 255, 256, 511, 512, 767, 768, M - 1) if c < M]
    top += [c for c in range(300, 312) if c < M and c not in top]
    top = sorted(set(top))
    bottom = [c for c in (3, 257, 770, M - 2) if 0 <= c < M and c not in top]
    return top, bottom


def _family_a(rng, M, dim, B, top, bottom):
    qh = rng.integers(-2, 3, (B, dim)) / 4.0
    ql = np.zeros((B, dim))
    a = _nonzero_a(rng, (M, dim))
    s = _sign(qh[0])
    a[top] = 2 * s                    # one hi row, each copy with its own lo row
    a[bottom] = -2 * s
    c = _lo_units(rng, a)
    return qh, ql, a / 4.0, c * LO_A


def _family_b(rng, M, dim, B, top, bottom):
    a = _nonzero_a(rng, (B, dim))
    c = _lo_units(rng, a)
    # query 0 always has column pairs with equal hi and different lo parts: (0, 1) and (2, 3) when dim >= 4
    a[0, :4] = (2, 2, -3, -3)[:dim]
    c[0, :4] = (3, -3, 2, -1)[:dim]
    e = rng.integers(-3, 4, (M, dim))
    # query 0's best rows: sign(q_hi) with one pair (c1, c2) moved by +-1 / -+1 each, which keeps q_hi.e_hi and moves
    # q_lo.e_hi by +-(q_lo[c1] - q_lo[c2])
    pairs = [(i, j) for i in range(min(dim, 64)) for j in range(i + 1, min(dim, 64))
             if a[0, i] == a[0, j] and c[0, i] != c[0, j]]
    base = _sign(a[0])
    rows = []
    for _ in top:
        r = base.copy()
        i, j = pairs[rng.integers(len(pairs))]
        d = rng.choice([-1, 1])
        r[i] += d
        r[j] -= d
        rows.append(r)
    if top:
        e[top] = np.array(rows)
    if bottom:
        e[bottom] = -np.array(rows[:len(bottom)])
    return a / 4.0, c * LO_A, e / 4.0, np.zeros((M, dim))


def _active_cols(rng, dim):
    """Two distinct columns of every 16-column group (the last group may be ragged; dim % 8 == 0)."""
    c1, c2 = [], []
    for g in range(0, dim, 16):
        i, j = rng.choice(np.arange(g, min(g + 16, dim)), 2, replace=False)
        c1.append(i)
        c2.append(j)
    return np.array(c1), np.array(c2)


def _family_c(rng, M, dim, B, top, bottom):
    c1, c2 = _active_cols(rng, dim)
    act = np.r_[c1, c2]
    s = rng.choice([-1, 1], dim)
    qh = np.zeros((B, dim))
    qh[:, act] = s[act]                                  # every query: the same hi pattern on the active columns
    ql = np.zeros((B, dim))
    ql[:, act] = rng.choice([-1, 1], (B, act.size)) * LO_C
    eh = rng.choice([-1, 1], (M, dim)).astype(np.float64)
    eh[:, c2] = -s[c1] * s[c2] * eh[:, c1]              # q_hi.e_hi = 0 in every group
    el = rng.choice([-1, 1], (M, dim)) * LO_C
    if top:
        # query 0's best row: e_hi[c1] along q_lo[c1], and q_hi.e_lo cancelling inside each group as well
        h = rng.choice([-1, 1], dim).astype(np.float64)
        h[c1] = np.sign(ql[0, c1])
        h[c2] = -s[c1] * s[c2] * h[c1]
        lo = rng.choice([-1, 1], dim) * LO_C
        lo[c1], lo[c2] = s[c1] * LO_C, -s[c2] * LO_C
        # the groups whose two lo.lo terms have the same sign: flipping both lo parts there moves lo.lo by 4 2^-20
        # and keeps every other term
        same = np.nonzero(ql[0, c1] * lo[c1] == ql[0, c2] * lo[c2])[0]
        rows = []
        for _ in top:
            r = lo.copy()
            if same.size:
                g = same[rng.random(same.size) < 0.5]
                r[c1[g]], r[c2[g]] = -r[c1[g]], -r[c2[g]]
            rows.append(r)
        eh[top] = h
        el[top] = np.array(rows)
        if bottom:
            eh[bottom] = -h
            el[bottom] = -np.array(rows[:len(bottom)])
    return qh, ql, eh, el


FAMILIES = {"A": _family_a, "B": _family_b, "C": _family_c}


def _stored(hi, lo):
    """float32 x = hi + lo, checked to split back into exactly this hi and lo."""
    x = (hi + lo).astype(np.float32)
    assert np.array_equal(x.astype(np.float64), hi + lo)
    h, l = _split(x)
    assert np.array_equal(h, hi) and np.array_equal(l, lo)
    return x


def make_case(family, M, dim, B, seed=0):
    rng = np.random.default_rng([ord(family), M, dim, B, seed])
    top, bottom = _planted_cols(M)
    qh, ql, eh, el = FAMILIES[family](rng, M, dim, B, top, bottom)
    if B > 128:
        qh[128], ql[128] = qh[0], ql[0]                  # the same planted rows in the second query tile
    return dict(family=family, Q=_stored(qh, ql), E=_stored(eh, el), qh=qh, ql=ql, eh=eh, el=el, top=top,
                bottom=bottom)


def exact_scores(qh, ql, eh, el):
    """(s4, s1): the float64 values of (q_hi + q_lo).(e_hi + e_lo) and q_hi.e_hi as float32, checked exact."""
    s4 = (qh + ql) @ (eh + el).T
    s1 = qh @ eh.T
    out = []
    for s in (s4, s1):
        f = s.astype(np.float32)
        assert np.array_equal(f.astype(np.float64), s)
        out.append(f)
    return out


def _quantum(case):
    return {"A": 2.0 ** -14, "B": 2.0 ** -14, "C": 2.0 ** -20}[case["family"]]


def significant_bits(case):
    """Bits from the largest partial sum a dot product can reach down to the quantum of its products.  A and B: any
    order of the four products of all columns (the larger of the positive and the negative sum).  C: the hi.hi
    products of one 16-column group are one +1 and one -1 (they enter the accumulator in one wgmma step), so a
    partial sum is at most the sum of |every other product| + 1."""
    qh, ql, eh, el = case["qh"], case["ql"], case["eh"], case["el"]
    terms = [(qh, eh), (qh, el), (ql, eh), (ql, el)]
    if case["family"] == "C":
        small = sum(np.abs(a) @ np.abs(b).T for a, b in terms[1:])
        reach = small + 1.0
    else:
        pos = sum(np.maximum(a, 0) @ np.maximum(b, 0).T + np.minimum(a, 0) @ np.minimum(b, 0).T for a, b in terms)
        neg = sum(np.maximum(a, 0) @ -np.minimum(b, 0).T + -np.minimum(a, 0) @ np.maximum(b, 0).T for a, b in terms)
        reach = np.maximum(pos, neg)
    units = reach / _quantum(case)
    return int(np.ceil(np.log2(units.max() + 1)))


# (M facts, dim, B queries): the M classes of STAGE_A_CASES around the 256-column tile and the 8-best list, dims with a
# ragged 16-column step (8, 24, 40, 136), multiples of 32 that are not of 64 (96, 160: the split stage is 32 columns
# wide, the bf16 stage 64), 768 and 1024; query counts around the 128-query tile
SPLIT_CASES = [
    (1, 8, 129), (9, 24, 128), (255, 40, 127), (257, 96, 129),
    (511, 136, 1), (513, 160, 128), (1003, 768, 129), (1003, 1024, 127),
]
CASE_IDS = [f"{fam}-M{M}-d{dim}-B{B}" for fam in "ABC" for M, dim, B in SPLIT_CASES]
CASES = [(fam, M, dim, B) for fam in "ABC" for M, dim, B in SPLIT_CASES]


# ------------------------------------------------------------------------------ defects of the mainloop, in numpy
def _shift16(x):
    """Column c read from column c ^ 16 inside its 32-column k-block; past dim the TMA fill is zero."""
    dim = x.shape[1]
    src = np.arange(dim) ^ 16
    out = np.zeros_like(x)
    ok = src < dim
    out[:, ok] = x[:, src[ok]]
    return out


def _ragged_zero(x):
    out = x.copy()
    out[:, x.shape[1] // 32 * 32:] = 0
    return out


def _row_off(x):
    out = np.zeros_like(x)
    out[:-1] = x[1:]
    return out


MUTATIONS = {
    "drop lo.lo": lambda qh, ql, eh, el: (None, "lolo"),
    "drop hi.lo": lambda qh, ql, eh, el: (None, "hilo"),
    "drop lo.hi": lambda qh, ql, eh, el: (None, "lohi"),
    "drop hi.hi": lambda qh, ql, eh, el: (None, "hihi"),
    "q_lo read from the hi plane": lambda qh, ql, eh, el: ((qh, qh, eh, el), None),
    "e_lo read from the hi plane": lambda qh, ql, eh, el: ((qh, ql, eh, eh), None),
    "q_hi read from the lo plane": lambda qh, ql, eh, el: ((ql, ql, eh, el), None),
    "e_hi read from the lo plane": lambda qh, ql, eh, el: ((qh, ql, el, el), None),
    "q_lo k-offset +16": lambda qh, ql, eh, el: ((qh, _shift16(ql), eh, el), None),
    "e_lo k-offset +16": lambda qh, ql, eh, el: ((qh, ql, eh, _shift16(el)), None),
    "ragged last k-block lo read as zero": lambda qh, ql, eh, el: ((qh, _ragged_zero(ql), eh, _ragged_zero(el)), None),
    "q_lo row off by one": lambda qh, ql, eh, el: ((qh, _row_off(ql), eh, el), None),
    "e_lo row off by one": lambda qh, ql, eh, el: ((qh, ql, eh, _row_off(el)), None),
}


def mutated_s4(case, name):
    """The split GEMM's scores with one defect, in float64 rounded to float32."""
    ops, drop = MUTATIONS[name](case["qh"], case["ql"], case["eh"], case["el"])
    qh, ql, eh, el = ops if ops is not None else (case["qh"], case["ql"], case["eh"], case["el"])
    prods = {"lolo": (ql, el), "hilo": (qh, el), "lohi": (ql, eh), "hihi": (qh, eh)}
    return sum(a @ b.T for p, (a, b) in prods.items() if p != drop).astype(np.float32)


def _selection_outputs(s, ks):
    norm, order = minmax32(s), ranking(s)
    return [expected_topk(norm, order, k)[:2] for k in ks]


def _differs(a, b):
    return any(not (np.array_equal(ia, ib) and np.array_equal(sa, sb)) for (ia, sa), (ib, sb) in zip(a, b))


# ------------------------------------------------------------------------------ CPU: the premises
@pytest.mark.parametrize("family", "ABC")
def test_split_premise_on_host(family):
    """Every generated row splits back into its intended hi and lo (make_case checks it), both planes are non-zero
    where the family says, every score is exact in float32, and every family stays within 22 significant bits:
    headroom against an adder that keeps fewer bits than fp32."""
    for M, dim, B in SPLIT_CASES:
        case = make_case(family, M, dim, B)
        s4, s1 = exact_scores(case["qh"], case["ql"], case["eh"], case["el"])
        assert (np.any(case["el"] != 0)) == (family in "AC") and (np.any(case["ql"] != 0)) == (family in "BC")
        assert significant_bits(case) <= 22, (family, M, dim, B, significant_bits(case))
        top = case["top"]
        if family in "AB" and len(top) > 1:
            assert np.all(s1[0, top] == s1[0, top[0]])                 # one hi row
            assert np.unique(s4[0, top]).size > 1                       # the lo rows decide
            if M > 311:
                assert np.all(s1[0, top] == s1[0].max())
                order = ranking(s4)[0]
                assert set(order[:8]) < set(top), (family, M, dim)      # the top-8 cut inside the planted rows
                assert ranking(s1)[0][:8].tolist() != order[:8].tolist()
        if family == "C":
            assert np.all(s1 == 0)                                      # q_hi.e_hi cancels in every group
            if len(top) > 1 and dim >= 768:
                lolo = case["ql"][0] @ case["el"][top].T
                cross = s4[0, top].astype(np.float64) - lolo
                assert np.unique(cross).size == 1 and np.unique(lolo).size > 1   # only lo.lo differs


def test_split_premise_values():
    """The families' boundary entries split as intended: a/4 + c 2^-12 with |c| = 3 at |a| >= 2 and |c| = 1 at
    |a| = 1 (below 0.25 the grid is finer), and +-1 -+ 2^-10."""
    a = np.array([2, -2, 3, -3, 1, -1, 1, -1], np.float64)
    c = np.array([-3, 3, -3, 3, -1, 1, 1, -1], np.float64)
    _stored(a / 4, c * LO_A)
    _stored(np.array([1.0, 1.0, -1.0, -1.0]), np.array([-1.0, 1.0, 1.0, -1.0]) * LO_C)
    # past half an ulp below the binade edge the split no longer gives this hi back (2 units are the tie, which rounds
    # to the even 0.25 and 1.0)
    h, _ = _split(np.array([0.25 - 2 * LO_A, 1 - 2 * LO_C, 0.25 - 3 * LO_A, 1 - 3 * LO_C], np.float32))
    assert h.tolist() == [0.25, 1.0, 0.25 - 2.0 ** -10, 1 - 2.0 ** -8]


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutations_change_the_expected_output(mutation):
    """For each defect, some case's expected output differs from what the defective kernel returns: the materialised
    scores, and the ids / min-max scores of the fused top-k (which reveals no raw score).  So the GPU tests below
    fail on each of these defects."""
    score_hit, fused_hit = [], []
    for fam, M, dim, B in CASES:
        case = make_case(fam, M, dim, B)
        s4, _ = exact_scores(case["qh"], case["ql"], case["eh"], case["el"])
        bad = mutated_s4(case, mutation)
        if not np.array_equal(bad, s4):
            score_hit.append((fam, M, dim, B))
            if _differs(_selection_outputs(bad, SMALL_K), _selection_outputs(s4, SMALL_K)):
                fused_hit.append((fam, M, dim, B))
    assert score_hit, f"{mutation}: no case's scores change"
    assert fused_hit, f"{mutation}: no case's fused top-k output changes"
    if mutation == "drop lo.lo":
        assert {c[0] for c in fused_hit} == {"C"}


# ------------------------------------------------------------------------------ GPU: the routes
@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def _threshold_outputs(s, thr, kmax):
    order = ranking(s)
    count = (s >= thr).sum(axis=1)
    ids, sc, _ = expected_topk(s, order, kmax)
    keep = np.arange(kmax)[None, :] < np.minimum(count, kmax)[:, None]
    return np.where(keep, ids, -1), np.where(keep, sc, np.float32(0)), count.astype(np.int32)


def check_split_routes(hb, e, Q, s4, s1, what, ks=SMALL_K + RADIX_K):
    """stage_a (fused and materialised, every k), the materialised score matrix, similarity and topk_similarity on
    the facts and the passages (both hold the same matrix), and knn_threshold at a planted score: all equal to
    numpy in both tensor-core modes."""
    try:
        for mode, s, name in ((hb.SIM_BF16X3, s4, "bf16x3"), (hb.SIM_BF16, s1, "bf16")):
            e.set_options(sim_mode=mode)
            norm, order = minmax32(s), ranking(s)
            for keep in (False, True):
                e.debug_keep_scores(keep)
                for k in ks:
                    idx, sc, nv = e.stage_a(Q, k)
                    want_idx, want_sc, want_nv = expected_topk(norm, order, k)
                    tag = f"{what} {name} keep={keep} k={k}"
                    assert_same(nv, want_nv, tag + ": n_valid")
                    assert_same(idx, want_idx, tag + ": ids")
                    assert_same(sc, want_sc, tag + ": scores")
                if keep:
                    got = e.debug_scores(0)
                    assert got.shape[0] > 0
                    assert_same(got, s[s.shape[0] - got.shape[0]:], f"{what} {name}: materialised scores")
            e.debug_keep_scores(False)
            for which in (0, 1):
                assert_same(e.similarity(which, Q), norm, f"{what} {name}: similarity({which})")
                for k in (1, 8, 33):
                    ids, sc = e.topk_similarity(which, Q, k)
                    want_ids, want_sc, _ = expected_topk(s, order, k)
                    assert_same(ids, want_ids, f"{what} {name}: topk_similarity({which}) k={k} ids")
                    assert_same(sc, want_sc, f"{what} {name}: topk_similarity({which}) k={k} scores")
            # the threshold: query 0's 6th best score, so the planted rows straddle it
            thr = s[0, order[0, min(5, s.shape[1] - 1)]]
            ids, sc, found = e.knn_threshold(0, Q, float(thr), 16)
            want_ids, want_sc, count = _threshold_outputs(s, thr, 16)
            assert_same(found, count, f"{what} {name}: knn_threshold n_found")
            ok = count <= 512                                     # rows past the candidate cap keep 512 of theirs
            assert_same(ids[ok], want_ids[ok], f"{what} {name}: knn_threshold ids")
            assert_same(sc[ok], want_sc[ok], f"{what} {name}: knn_threshold scores")
    finally:
        e.debug_keep_scores(False)
        e.set_options(sim_mode=hb.SIM_BF16X3)


@pytest.mark.gpu
@pytest.mark.parametrize("family,M,dim,B", CASES, ids=CASE_IDS)
def test_split_routes_exact(hb, family, M, dim, B):
    case = make_case(family, M, dim, B)
    s4, s1 = exact_scores(case["qh"], case["ql"], case["eh"], case["el"])
    e = hb.Engine(0)
    try:
        e.load_embeddings(case["E"], case["E"])
        check_split_routes(hb, e, case["Q"], s4, s1, f"{family} M={M} dim={dim} B={B}")
    finally:
        e.close()


# ------------------------------------------------------------------------------ GPU: the screen and the placements
F_SCREEN = 65_536 + 37          # screened (>= 65,536 facts), not a multiple of the 256-fact tile
D_SCREEN = 224                  # a multiple of 32, not of 64: ragged against the 64-column hi-only stage
B_SCREEN = 130


def _err_bound64(qh, ql, eh, el, gain=1.0):
    """E_q of DESIGN.md section 4, K2, in float64 without the (1 + 2^-10) rounding factor; `gain` scales its
    accumulation term."""
    Hf, Lf = np.linalg.norm(eh, axis=1).max(), np.linalg.norm(el, axis=1).max()
    nh, nl = np.linalg.norm(qh, axis=1), np.linalg.norm(ql, axis=1)
    steps = 5 * -(-qh.shape[1] // 16)
    return nh * Lf + nl * Hf + nl * Lf + gain * steps * ACC_STEP * (nh + nl) * (Hf + Lf)


def screen_case():
    """Family A at F_SCREEN x 768 with B_SCREEN queries.  Every query has 12 planted best rows (one hi row, 12 lo rows)
    with at most 7 in one tile and 3 planted worst rows in 3 tiles, at random rows; query 0's are at the columns of
    _planted_cols (query 128 is its copy).  So each query's top 8 and minimum are decided by lo, the screen's
    candidate bands hold exactly its planted rows, no tile is saturated and no cap is reached."""
    rng = np.random.default_rng(31)
    M, dim, B = F_SCREEN, D_SCREEN, B_SCREEN
    top0, bottom0 = _planted_cols(M)
    qh, _, eh, el = _family_a(rng, M, dim, B, top0, bottom0)
    qh[128] = qh[0]
    a = eh * 4
    free = np.setdiff1d(np.arange(M), top0 + bottom0)
    picks = rng.choice(free, (B, 15), replace=False)
    tops, bottoms = [top0], [bottom0]
    for b in range(1, B):
        if b == 128:
            tops.append(top0)
            bottoms.append(bottom0)
            continue
        t, lo = np.sort(picks[b, :12]), np.sort(picks[b, 12:])
        s = _sign(qh[b])
        a[t] = 2 * s
        a[lo] = -2 * s
        tops.append(list(t))
        bottoms.append(list(lo))
    c = _lo_units(rng, a)
    eh, el = a / 4.0, c * LO_A
    ql = np.zeros_like(qh)
    return dict(family="A", Q=_stored(qh, ql), E=_stored(eh, el), qh=qh, ql=ql, eh=eh, el=el, tops=tops,
                bottoms=bottoms)


@pytest.fixture(scope="module")
def screened():
    case = screen_case()
    s4, s1 = exact_scores(case["qh"], case["ql"], case["eh"], case["el"])
    case.update(s4=s4, s1=s1)
    return case


def test_screen_case_premise(screened):
    """The screen case's design, checked in numpy: the bands L - 2 E_q and U + 2 E_q of every query hold exactly its
    planted rows, lo decides each query's top 8 and minimum, and the screen's caps hold -- at most 256 listed
    candidates and 8 saturated tiles per query (a tile whose list's 8th key, or whose second smallest, lies in a band)
    and at most 48 staged tiles per 128-query m-tile (one per candidate row sharing a column f mod 256), as the model
    of test_gpu_screen_caps counts them -- so no chunk should fall back."""
    from tests.test_gpu_screen_caps import screen_bound, screen_model
    c = screened
    s4, s1 = c["s4"].astype(np.float64), c["s1"].astype(np.float64)
    E = screen_bound(c["qh"], c["ql"], c["eh"], c["el"])
    assert significant_bits(c) <= 22
    model = screen_model(c["s1"], c["s4"], E, np.arange(B_SCREEN))
    for b in range(B_SCREEN):
        top, bottom = c["tops"][b], c["bottoms"][b]
        acc = model["acc"][b]
        assert set(np.nonzero(s1[b] >= acc["L"] - 2 * E[b])[0]) == set(top), b
        assert set(np.nonzero(s1[b] <= acc["U"] + 2 * E[b])[0]) == set(bottom), b
        assert np.all(s1[b, top] == s1[b, top[0]]) and np.all(s1[b, bottom] == s1[b, bottom[0]])
        assert np.unique(s4[b, top]).size > 4 and np.unique(s4[b, bottom]).size > 1
        assert acc["n"] <= 256 and len(acc["sat"]) <= 8
        if b in (0, 128):
            assert acc["sat"] == [1]                            # query 0's 14 rows in tile 1
    assert max(ch["max_col"] for ch in model["chunks"]) <= 48 and model["fallbacks"] == 0


def _assert_stage_a_exact(e, case, ks, what, fallbacks=0, minmax=True):
    Q, s = case["Q"], case["s4"]
    norm, order = minmax32(s), ranking(s)
    for k in ks:
        e.reset_stats()
        idx, sc, nv = e.stage_a(Q, k)
        fb = e.stats()["stage_a_fallbacks"]
        want_idx, want_sc, want_nv = expected_topk(norm, order, k)
        tag = f"{what} k={k}"
        assert_same(nv, want_nv, tag + ": n_valid")
        assert_same(idx, want_idx, tag + ": ids")
        assert_same(sc, want_sc, tag + ": scores")
        if minmax and k <= 8:
            mm = np.stack([s.min(axis=1), s.max(axis=1)], axis=1)
            assert_same(e.debug_fact_minmax(), mm, tag + ": mm_fact")
        if fallbacks is not None and k <= 8:
            assert fb == fallbacks, f"{tag}: {fb} fallbacks, designed for {fallbacks}"


@pytest.mark.gpu
def test_screen_lo_decides_exact(hb, screened):
    """The screened stage A (and the exact path on the same handle) against numpy, with each query's top 8 and minimum
    decided by its lo rows; the case keeps every cap, so no chunk falls back."""
    e = hb.Engine(0)
    try:
        e.load_embeddings(screened["E"], screened["E"][:4])
        _assert_stage_a_exact(e, screened, SMALL_K, "screened")
        e.debug_exact_stage_a(True)
        try:
            _assert_stage_a_exact(e, screened, (1, 8), "exact path")
        finally:
            e.debug_exact_stage_a(False)
    finally:
        e.close()


def _lo_budget(rows, dim):
    """The hi plane plus two 256-row lo slices."""
    return rows * dim * 2 + 2 * 256 * dim * 2 + 100


def _tiny_graph_engine(hb, fe, pe):
    """A mutable handle over two entities and one vertex per passage (append and delete need a graph and tables)."""
    F, P = fe.shape[0], pe.shape[0]
    n = 2 + P
    pv = np.arange(2, n, dtype=np.int32)
    e = hb.Engine(0, mutable=True)
    e.load_graph(n, pv, np.zeros(P, np.int32), np.ones(P))
    e.load_tables(pv, np.zeros(F, np.int32), np.ones(F, np.int32), np.r_[1, 1, np.zeros(P)].astype(np.int32))
    e.load_embeddings(fe, pe)
    return e


def _append_rows(e, fe, pe):
    n0, F, P = e.n_nodes, fe.shape[0], pe.shape[0]
    pv = np.arange(n0, n0 + P, dtype=np.int32)
    cc = np.r_[1, 1, np.zeros(n0 + P - 2)].astype(np.int32)
    e.append(P, pv, np.zeros(P, np.int32), np.ones(P), pv, np.zeros(F, np.int32), np.ones(F, np.int32), cc,
             fe, pe if P else None)


def _placed_engine(hb, layout, fe, pe, cut):
    """fe (and pe) loaded whole, streamed in three chunks, as rows [:cut] plus an append of the rest, under a device
    budget that puts both fact planes in pinned host memory, or with the lo plane alone there."""
    F, dim = fe.shape
    if layout == "whole":
        e = hb.Engine(0)
        e.load_embeddings(fe, pe)
    elif layout == "streamed":
        e = hb.Engine(0)
        for which, m in ((0, fe), (1, pe)):
            r = m.shape[0]
            e.load_embeddings_streamed(which, r, dim, [(0, m[:r // 3]), (r // 3, m[r // 3:r - 5]), (r - 5, m[r - 5:])])
        e.n_passages = pe.shape[0]
    elif layout == "appended":
        e = _tiny_graph_engine(hb, fe[:cut], pe[:max(1, pe.shape[0] // 2)])
        _append_rows(e, fe[cut:], pe[max(1, pe.shape[0] // 2):])
    elif layout == "host planes":
        e = hb.Engine(0, fact_device_bytes=2 * (-(-F // 4 // 256) * 256) * dim * 4 + 1000)
        e.load_embeddings(fe, pe)
        assert e.fact_planes_info()["on_host"] == 1
    else:
        e = hb.Engine(0, fact_device_bytes=_lo_budget(F, dim), fact_lo_on_host=True)
        e.load_embeddings(fe, pe)
        assert e.fact_planes_info()["on_host"] == 2
    return e


PLACEMENTS = ["whole", "streamed", "appended", "host planes", "lo on host"]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", PLACEMENTS)
def test_screen_case_placements(hb, screened, layout):
    """The screen case under every placement of the fact planes, each against numpy (not against another
    placement): the fused top-k (screened where the planes allow) and the radix route."""
    fe = screened["E"]
    e = _placed_engine(hb, layout, fe, fe[:300], cut=F_SCREEN - 1000)
    try:
        _assert_stage_a_exact(e, screened, (1, 5, 8, 9, 32), layout, minmax=layout != "host planes")
    finally:
        e.close()


# ------------------------------------------------------------------------------ GPU: the planes against the numpy split
def _bits(x):
    return np.ascontiguousarray(x, np.float32).view(np.uint32)


def special_values():
    """float32 bit patterns where a bf16 split goes wrong, with what the split must give (hi, lo as bf16 bits)."""
    v = np.array([
        0x3F808000, 0x3F818000, 0xBF808000, 0xBF818000,   # halfway ties: even neighbour (down), odd neighbour (up)
        0x40A08000, 0x40A18000,
        0x3FFFFFFF, 0x3FFF8000, 0xBFFFC000, 0x7EFFFFFF,   # hi rounds up into the next binade
        0x00000000, 0x80000000,                           # +0, -0
        0x00000001, 0x807FFFFF, 0x00012345, 0x00008000,   # subnormals (and a subnormal tie)
        0x00018000, 0x80010001,
        0x7F7F7FFF,                                       # the largest float32 whose hi stays finite
        0x3EAAAAAB, 0xC0490FDB,                           # ordinary values
    ], np.uint32)
    return v.view(np.float32)


def _split_bits(x):
    hi = _bf16(x)
    with np.errstate(over="ignore", invalid="ignore"):
        lo = _bf16(np.asarray(x, np.float32) - hi)
    return (_bits(hi) >> 16).astype(np.uint16), (_bits(lo) >> 16).astype(np.uint16)


def test_special_value_split_on_host():
    """What the planes must hold for the special values (the numpy split the GPU planes are compared with)."""
    hi, lo = _split_bits(special_values())
    assert hi[:6].tolist() == [0x3F80, 0x3F82, 0xBF80, 0xBF82, 0x40A0, 0x40A2]
    assert lo[0] == 0x3B80 and lo[1] == 0xBB80                       # +-2^-8 . 2^0 ... the half ulp, either sign
    assert hi[6:10].tolist() == [0x4000, 0x4000, 0xC000, 0x7F00]
    assert hi[10:12].tolist() == [0x0000, 0x8000] and lo[10:12].tolist() == [0, 0]
    # subnormals are rounded, not flushed: 0x00012345 keeps a subnormal hi, 0x807FFFFF rounds up to the smallest
    # normal, the subnormal tie 0x00018000 rounds to the even 0x0002, and 0x80010001 leaves lo = -0
    assert hi[14] == 0x0001 and hi[13] == 0x8080 and hi[16] == 0x0002
    assert hi[17] == 0x8001 and lo[17] == 0x8000
    assert hi[18] == 0x7F7F and lo[18] != 0
    # near FLT_MAX the hi part rounds to +inf and lo = x - inf = -inf
    big = np.array([np.finfo(np.float32).max], np.float32)
    bh, bl = _split_bits(big)
    assert bh[0] == 0x7F80 and bl[0] == 0xFF80


def _plane_matrix(rng, rows, dim):
    """Family A rows with the special values spread over rows and columns (the last 4-column group included)."""
    x = (_nonzero_a(rng, (rows, dim)) / 4.0 + _lo_units(rng, np.ones((rows, dim), int) * 2) * LO_A).astype(np.float32)
    v = special_values()
    for i, val in enumerate(v):
        x[(7 * i) % rows, (13 * i) % dim] = val
        x[(rows - 1 - i) % rows, dim - 1 - i % 4] = val
    return x


def _assert_planes(e, fe, pe, what):
    for which, m in (("fact", fe), ("passage", pe)):
        want_hi, want_lo = _split_bits(m)
        assert_same(e.debug_index(f"{which}_hi"), want_hi, f"{what}: {which}_hi")
        assert_same(e.debug_index(f"{which}_lo"), want_lo, f"{what}: {which}_lo")


@pytest.mark.gpu
@pytest.mark.parametrize("dim", [40, 96])
def test_planes_equal_numpy_split(hb, dim):
    rng = np.random.default_rng(dim)
    fe, pe = _plane_matrix(rng, 1003, dim), _plane_matrix(rng, 301, dim)
    for layout in ("whole", "streamed", "appended"):
        e = _placed_engine(hb, layout, fe, pe, cut=600)
        try:
            _assert_planes(e, fe, pe, f"{layout} dim={dim}")
        finally:
            e.close()


@pytest.mark.gpu
def test_screen_falls_back_on_an_infinite_hi(hb, screened):
    """A fact entry near FLT_MAX has hi = +inf and lo = -inf: the plane norm is +inf, E_q is not finite, and every
    screened chunk falls back to the exact path, which the stats count."""
    fe = screened["E"].copy()
    fe[1000, 7] = np.finfo(np.float32).max
    e = hb.Engine(0)
    try:
        e.load_embeddings(fe, fe[:4])
        row = e.debug_index("fact_hi")[1000]
        assert row[7] == 0x7F80 and e.debug_index("fact_lo")[1000, 7] == 0xFF80
        e.reset_stats()
        e.stage_a(screened["Q"], 8)
        assert e.stats()["stage_a_fallbacks"] == 1
    finally:
        e.close()


# ------------------------------------------------------------------------------ GPU: the accumulation premise under E_q
def _premise_inputs():
    """(name, facts, queries) float32: C3-shaped unit vectors, near-duplicates, and rows built against adders that
    align their addends to the accumulator and truncate."""
    out = []
    for dim in (768, 1024):
        rng = np.random.default_rng(dim)
        fe = _unit(rng.standard_normal((4096, dim)))
        base = fe[rng.integers(0, 4096, 512)]
        out.append((f"unit d={dim}", fe, _unit(base + 0.5 * rng.standard_normal(base.shape) / np.sqrt(dim))))
    rng = np.random.default_rng(3)
    fe = _unit(rng.standard_normal((4096, 768)))
    out.append(("near-duplicates d=768", fe, _unit(fe[:512] + 1e-4 * rng.standard_normal((512, 768)))))
    dim = 768
    # products of the later columns at 2^-23 (1 - 2^-8), 2^-24, 2^-25 and 2^-26 of the first, all positive; then
    # products just below 2^-24 and 1.5 2^-24 (13 and 3 of each 16 columns), which an adder that keeps two bits below
    # the accumulator's last and truncates each addend nearly loses by 2^-25 each, with the kept parts summing to
    # 19 2^-25 per step, off the fp32 grid; the last variant has lo parts (2^-12 (1 + 2^-9) splits into 2^-12 + 2^-21)
    below = np.where(np.arange(768) % 16 < 13, 1 - 2.0 ** -8, 1.5 - 2.0 ** -7) * 2.0 ** -12
    smalls = [2.0 ** -11 * (1 - 2.0 ** -8), 2.0 ** -12, 2.0 ** -13, 2.0 ** -14, below, 2.0 ** -12 * (1 + 2.0 ** -9)]
    q_small = [2.0 ** -12, 2.0 ** -12 * (1 + 2.0 ** -9)]
    for name, big in (("big-first parallel rows", np.arange(dim) == 0),
                      ("one large and fifteen small products per k16 group", np.arange(dim) % 16 == 0)):
        fe = np.stack([np.where(big, 1.0, v) for v in smalls for _ in range(64)]).astype(np.float32)
        Q = np.stack([np.where(big, 1.0, v) for v in q_small]).astype(np.float32)
        out.append((name, fe, Q))
    # large cancelling pairs (+1 . 1, 1 . -1) at the head of every k16 group, then small products
    pair = np.arange(dim) % 16
    fe = np.stack([np.where(pair == 0, 1.0, np.where(pair == 1, -1.0, v)) for v in smalls for _ in range(64)])
    Q = np.stack([np.where(pair < 2, 1.0, v) for v in q_small])
    out.append(("cancelling pairs then a small remainder", fe.astype(np.float32), Q.astype(np.float32)))
    # the sign-aligned lo rows of test_screen_sign_aligned_lo_parts: |s4 - s1| near E_q
    rng = np.random.default_rng(11)
    B, per = 128, 24
    signs = rng.choice([-1.0, 1.0], (B, dim))
    rows = np.repeat(signs, per, axis=0)
    rho = rng.choice([-1.0, 1.0], (B * per, 1)) * rows
    pad = rng.choice([-1.0, 1.0], (1000, dim))
    fe = np.concatenate([_aligned(rng, rows, rho), _aligned(rng, pad, rng.choice([-1.0, 1.0], pad.shape))])
    out.append(("sign-aligned lo parts", fe, _aligned(rng, signs, signs)))
    return out


def _materialised(hb, e, Q, mode):
    e.set_options(sim_mode=mode)
    e.debug_keep_scores(True)
    e.stage_a(Q, 1)
    S = e.debug_scores(0).astype(np.float64)
    assert S.shape == (Q.shape[0], e.n_facts)
    return S


@pytest.mark.gpu
def test_accumulation_within_the_screen_model(hb):
    """Per GEMM: |score - the float64 value of its own bf16 products| <= steps ACC_STEP sum|products|, steps = d/16
    for hi.hi (the screen's s1) and 4 d/16 for the split product (s4), on every pair.  Per pair: |s4 - s1| <= E_q of
    DESIGN.md section 4, K2, without its (1 + 2^-10) rounding factor.  The largest error / model ratio of each input
    is printed and named in any failure.  (The big-first rows with products just below 2^-24 and 1.5 2^-24 lose
    19 2^-25 per step on the H100: 1.18 times the 2^-21 the bound assumed before.)"""
    report, failures = [], []
    for name, fe, Q in _premise_inputs():
        dim = fe.shape[1]
        qh, ql = _split(Q)
        eh, el = _split(fe)
        e = hb.Engine(0)
        try:
            e.load_embeddings(fe, fe[:4])
            s1 = _materialised(hb, e, Q, hb.SIM_BF16)
            s4 = _materialised(hb, e, Q, hb.SIM_BF16X3)
        finally:
            e.close()
        steps = -(-dim // 16)
        exact1, abs1 = qh @ eh.T, np.abs(qh) @ np.abs(eh).T
        exact4, abs4 = (qh + ql) @ (eh + el).T, (np.abs(qh) + np.abs(ql)) @ (np.abs(eh) + np.abs(el)).T
        with np.errstate(divide="ignore", invalid="ignore"):
            r1 = np.nan_to_num(np.abs(s1 - exact1) / (steps * ACC_STEP * abs1))
            r4 = np.nan_to_num(np.abs(s4 - exact4) / (4 * steps * ACC_STEP * abs4))
            rq = np.abs(s4 - s1) / _err_bound64(qh, ql, eh, el)[:, None]
        worst = {"hi.hi": float(r1.max()), "split": float(r4.max()), "|s4 - s1| / E_q": float(rq.max())}
        report.append(f"{name}: " + ", ".join(f"{k} {v:.4g}" for k, v in worst.items()))
        if max(worst.values()) > 1:
            failures.append(report[-1])
    print("\nerror / model ratios (largest over all pairs):\n  " + "\n  ".join(report))
    assert not failures, "accumulation outside the screen's model: " + "; ".join(failures)
