"""PPR sweeps on exact arithmetic: the fp32 sweep (K1) and the fp16 sweep (K1m) against float64, bit for bit.

The kernels do not need P to be stochastic, so the CSR is loaded directly with every value a power of two (2^-1 ...
2^-6), the damping is 0.5 and the reset vectors are small integers.  Every product is then dyadic; when, for every row,
sum_j |a P_ij x_j| + |v_i| fits in 24 bits above the finest term (the premise, checked on the host below), every partial
sum of the row in ANY order is an exact float32, so the result does not depend on how a kernel orders its sums and
equality is the right test.  The same holds for the column sums (checked per 256-row block and over the long rows, the
most a CTA ever adds) and, for the fp16 solver, for every stored iterate (exactly representable in fp16, never clamped).

Row structure: lengths 0..9 (the ragged predicated batch of K1m, the scalar tail of K1), 255 / 256 / 257 / 511 / 512 /
513 and a hub of 5,000 around the 256-non-zero long-row cut (segments, fixed-order finalize, more than 64 long rows so a
second finalize CTA runs), self-loops, isolated vertices, n_rows of 1, 63, 64, 65 and 4,133, and 64-row blocks that mix
long and short rows so row_order really permutes.  Long rows gather mostly from "dead" vertices (empty row, v = 0) and
from leaves (empty row, integer v), which keeps their sums small; edges into rows that are not leaves carry 2^-1 or
2^-2, which keeps the granularity of an iterate coarse enough for three sweeps.

Chebyshev steps (w != 1) cannot be exact: they are compared per entry with a float64 emulation of the same truncated
recurrence, with a tolerance derived from the storage precision.  Stage B's compact right-hand side is compared with the
dense path of hrag_ppr bit for bit, and every column of a sweep must be independent of the others.
"""
import numpy as np
import pytest

ALPHA = 0.5
T = 64.0                     # kMixedT: the residual of the refinement round is stored times 64
SHORT = (0, 1, 2, 3, 4, 5, 7, 8, 9)
LONG = (255, 256, 257, 511, 512, 513)
HUB = 5000


# ------------------------------------------------------------------------------ fixtures
class Graph:
    def __init__(self, n, row_ptr, col, val, leaf, dead, probes):
        self.n, self.row_ptr, self.col, self.val = n, row_ptr, col, val
        self.leaf, self.dead, self.probes = leaf, dead, probes
        self.iso = np.zeros(0, np.int64)
        import scipy.sparse as sp
        # copies: scipy shares index arrays and may sort them in place, which would scramble the CSR the engine loads
        self.P = sp.csr_matrix((val.astype(np.float64), col.copy(), row_ptr.copy()), shape=(n, n))
        self.lengths = np.diff(row_ptr)
        self.long = np.nonzero(self.lengths > 256)[0]


def _planted(L):
    """CSR positions inside a row of length L that a few-hot column probes: first, last, 4k + 3, 255, 256 and the
    last element of a ragged last 256-segment."""
    pos = {0, L - 1, 3 if L > 3 else L - 1}
    if L > 256:
        pos |= {255, 256, 4 * (L // 8) + 3}
    return sorted(p for p in pos if 0 <= p < L)


def exact_graph(n, seed, extra_lengths=(), n_long_extra=0):
    """A CSR on n vertices with power-of-two values.  Row lengths: SHORT at random, plus extra_lengths and
    n_long_extra rows of 257..300 at random row positions.  Returns a Graph; probes = [(row, pos, leaf)] planted gather
    positions, each pointing at a leaf of its own that nothing else gathers."""
    rng = np.random.default_rng(seed)
    lengths = rng.choice(SHORT, size=n)
    lengths[rng.random(n) < 0.25] = 0                      # enough empty rows for dead vertices and leaves
    special = list(extra_lengths) + list(rng.integers(257, 301, n_long_extra))
    where = rng.permutation(n)[:len(special)] if n > 1 else np.zeros(len(special), np.int64)
    for r, L in zip(where, special):
        lengths[r] = L
    # every row of length 0 is a leaf or dead; make sure both kinds exist when the graph is big enough
    empty = np.nonzero(lengths == 0)[0]
    dead = np.zeros(n, bool)
    dead[empty[::2]] = True
    leaf = (lengths == 0) & ~dead
    iso = np.nonzero(leaf)[0][-1:] if n > 1 else np.zeros(0, np.int64)
    live = np.setdiff1d(np.nonzero(~dead)[0], iso)         # iso: a leaf nothing gathers (ballast of few-hot columns)
    plain_leaves = np.setdiff1d(np.nonzero(leaf)[0], iso)
    probe_rows = [r for r in range(n) if lengths[r] > 0 and (lengths[r] not in (4, 8) or lengths[r] > 256)]
    # probe leaves: one leaf per planted position, gathered nowhere else
    probes = []
    probe_leaf_pool = list(plain_leaves[len(plain_leaves) // 2:])
    rows, vals = {}, {}
    for r in range(n):
        L = int(lengths[r])
        if L == 0:
            continue
        c = np.empty(L, np.int64)
        v = np.empty(L, np.float32)
        for k in range(L):
            if L <= 9:
                pick_live = rng.random() < 0.8 or not dead.any()
                pool = live if pick_live else np.nonzero(dead)[0]
            else:
                pool = plain_leaves[:len(plain_leaves) // 2] if (rng.random() < 1 / 32 and len(plain_leaves) > 1) \
                    else np.nonzero(dead)[0]
                if len(pool) == 0:
                    pool = live
            j = int(rng.choice(pool))
            c[k] = j
            coarse = lengths[j] > 0
            v[k] = np.float32(2.0 ** -(rng.integers(1, 3) if coarse else rng.integers(1, 7)))
        if L <= 9 and rng.random() < 0.1:
            c[rng.integers(0, L)] = r                        # self-loop
            v[c == r] = np.float32(0.5)
        rows[r], vals[r] = c, v
    # planted probes, in priority order: one row of every listed length (longest first), the long rows that the second
    # long-row finalize CTA of K1m handles (long rows 64, 65, ...), then the others
    long_rows = [r for r in range(n) if lengths[r] > 256]
    firsts = [min(r for r in probe_rows if lengths[r] == L) for L in (HUB,) + LONG[::-1] + SHORT[::-1]
              if any(lengths[r] == L for r in probe_rows)]
    order = list(dict.fromkeys(firsts + long_rows[64:] + sorted(probe_rows, key=lambda r: -lengths[r])))
    for r in order:
        for p in _planted(int(lengths[r])):
            if not probe_leaf_pool:
                break
            u = int(probe_leaf_pool.pop())
            rows[r][p], vals[r][p] = u, np.float32(2.0 ** -rng.integers(1, 7))
            probes.append((r, p, u))
    kept = [r for r in range(n) if lengths[r] > 0]
    col = np.concatenate([rows[r] for r in kept]).astype(np.int32) if kept else np.zeros(0, np.int32)
    val = np.concatenate([vals[r] for r in kept]).astype(np.float32) if kept else np.zeros(0, np.float32)
    row_ptr = np.concatenate([[0], np.cumsum(lengths)]).astype(np.int64)
    g = Graph(n, row_ptr, col, val, leaf, dead, probes)
    g.iso = iso
    return g


def small_graph(n, seed, extra):
    """n in {63, 64, 65}: every class of n_rows around a 64-row block; columns may repeat inside a row."""
    return exact_graph(n, seed, extra)


def one_vertex_graph():
    """n = 1: two self-loops of 2^-3 (a row sum of 2^-1 would overflow the fp16 residual at (1, 1))."""
    return Graph(1, np.array([0, 2], np.int64), np.zeros(2, np.int32), np.array([2 ** -3, 2 ** -3], np.float32),
                 np.zeros(1, bool), np.zeros(1, bool), [])


GRAPHS = {
    "n1": one_vertex_graph,
    "n63": lambda: small_graph(63, 2, (513,)),
    "n64": lambda: small_graph(64, 5, (255, 256, 257)),
    "n65": lambda: small_graph(65, 5, (HUB, 511)),
    "n4133": lambda: exact_graph(4133, 5, LONG + (HUB,), n_long_extra=70),
}
_CACHE = {}


def graph(name):
    if name not in _CACHE:
        _CACHE[name] = GRAPHS[name]()
    return _CACHE[name]


def dense_reset(g, B, seed):
    """fp32 solver: dense columns of small integers (0 on dead vertices)."""
    rng = np.random.default_rng(seed)
    V = rng.integers(0, 4, size=(g.n, B)).astype(np.float64)
    V[g.dead] = 0
    V[:, V.sum(axis=0) == 0] = 1                           # no all-zero column
    return V


def fewhot_reset(g, B, seed):
    """fp16 solver: column b is one probe leaf (value 1..3) plus, on every third column, a second probe leaf; each
    column thereby exercises the gathers at its probes' planted CSR positions.  Weight 12 on a vertex nothing gathers
    lowers the column scale so that the (1, 1) residual 64 (aP)^2 s v stays inside fp16's range."""
    rng = np.random.default_rng(seed)
    V = np.zeros((g.n, B))
    if not g.probes:
        V[0] = 1
        return V
    for b in range(B):
        V[g.probes[b % len(g.probes)][2], b] = rng.integers(1, 4)
        if b % 3 == 2:
            V[g.probes[(7 * b + 1) % len(g.probes)][2], b] += 1
    V[g.iso] = 12
    return V


# ------------------------------------------------------------------------------ the exactness premise
def low_exp(a):
    """Exponent of the lowest set bit of every non-zero float64 (a large number for zeros: no constraint)."""
    a = np.asarray(a, np.float64)
    out = np.full(a.shape, 10_000, np.int64)
    nz = a != 0
    m, e = np.frexp(np.abs(a[nz]))
    mi = (m * 2.0 ** 53).astype(np.int64)
    out[nz] = e - 53 + np.log2((mi & -mi).astype(np.float64)).astype(np.int64)
    return out


def _fits(bound, lowexp, bits, what):
    """Every dyadic partial sum of magnitude <= bound on a 2^lowexp grid is exact with `bits` significant bits."""
    lowexp = np.minimum(lowexp, 900)
    ok = (bound == 0) | (bound < np.exp2(lowexp + float(bits)))
    assert np.all(ok), f"{what}: {np.count_nonzero(~ok)} sums exceed {bits} bits"
    assert np.all((bound == 0) | (lowexp >= -126)), f"{what}: below the float32 normal range"


def _row_min(g, a):
    """Per row (and column) minimum of a [nnz, B] array; rows without non-zeros -> 10_000."""
    out = np.full((g.n, a.shape[1]), 10_000, np.int64)
    ne = np.nonzero(g.lengths > 0)[0]
    if len(ne):
        out[ne] = np.minimum.reduceat(a, g.row_ptr[ne], axis=0)
    return out


def checked_sweep(g, X, add, scale_acc=ALPHA, what="sweep"):
    """y = scale_acc * P X + add in float64, after asserting the premise for every row: all partial sums of the row
    (bounded by sum_j |scale_acc P_ij X_j| + |add_i|) are exact float32 values."""
    terms = scale_acc * g.val.astype(np.float64)[:, None] * X[g.col]
    bound = np.abs(g.P) @ np.abs(X) * scale_acc + np.abs(add)
    _fits(bound, np.minimum(_row_min(g, low_exp(terms)), low_exp(add)), 24, what)
    return scale_acc * (g.P @ X) + add


def checked_colsum(g, Z, what):
    """Column sums of Z, after asserting that every CTA partial is exact: every 256-row block and the long rows."""
    blocks = [np.arange(b, min(g.n, b + 256)) for b in range(0, g.n, 256)] + [g.long]
    for rows in blocks:
        if len(rows):
            _fits(np.abs(Z[rows]).sum(axis=0), low_exp(Z[rows]).min(axis=0), 24, what + " column sum")
    return Z.sum(axis=0)


def assert_fp16(X, what):
    """Every stored fp16 value is exactly representable and is not clamped by sat_h (|x| <= 65504)."""
    assert np.all(np.abs(X) <= 65504), f"{what}: {np.count_nonzero(np.abs(X) > 65504)} values would be clamped"
    assert np.array_equal(X.astype(np.float16).astype(np.float64), X), f"{what}: not exact in fp16"


def fp32_power_expected(g, V, iters):
    """K1, PPR_POWER, `iters` sweeps from x = v: z = sum_{t <= iters} (aP)^t v; scores = fl32(z) / fl32(sum z)."""
    x = V
    for it in range(iters):
        x = checked_sweep(g, x, V, what=f"fp32 sweep {it + 1}")
    assert np.array_equal(x.astype(np.float32), x)
    s = checked_colsum(g, x, "fp32")
    return (x.astype(np.float32) / s.astype(np.float32)).T


def column_scale(vsum):
    """column_scale() of ppr_mixed.cu at damping 0.5: 2^floor(log2(32768 * 0.5 / sum v)), 1 for an empty column."""
    vs = np.asarray(vsum, np.float32)
    with np.errstate(divide="ignore"):
        sc = np.exp2(np.floor(np.log2(np.float32(16384.0) / vs))).astype(np.float32)
    return np.where(vs > 0, sc, np.float32(1)).astype(np.float64)


def mixed_11_expected(g, V):
    """K1m at mixed_sweeps (1, 1): x0 = aP sv + sv, r = 64 (sv - x0 + aP x0) (MODE 1), d = aP r + r, every one an exact
    fp16 value; x0 + d / 64 = s sum_{t<4} (aP)^t v.  Scores = fl32(x0 + d/64) / fl32(sum x0 + sum d / 64)."""
    B = V.shape[1]
    Vp = np.zeros((g.n, 32 * ((B + 31) // 32)))
    Vp[:, :B] = V
    out = np.empty((B, g.n), np.float32)
    for q0 in range(0, B, 32):
        v = Vp[:, q0:q0 + 32]
        s = column_scale(v.sum(axis=0))
        sv = v * s
        assert_fp16(sv, "rhs16")
        x0 = checked_sweep(g, sv, sv, what="x0")
        assert_fp16(x0, "x0")
        r = T * checked_sweep(g, x0, sv - x0, what="residual")
        assert_fp16(r, "r")
        d = checked_sweep(g, r, r, what="d")
        assert_fp16(d, "d")
        z = x0 + d / T
        assert np.array_equal(z.astype(np.float32), z)
        series = sv.copy()
        term = sv
        for _ in range(3):
            term = ALPHA * (g.P @ term)
            series = series + term
        assert np.array_equal(z, series)                   # what the (1, 1) solve computes, in closed form
        tot = checked_colsum(g, x0, "x0") + checked_colsum(g, d, "d") / T
        nb = min(32, B - q0)
        out[q0:q0 + nb] = (z[:, :nb].astype(np.float32) / tot[:nb].astype(np.float32)).T
    return out


FP32_WIDTHS = (4, 8, 16, 32, 64)


# ------------------------------------------------------------------------------ CPU: the premise itself
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_exact_premise_on_host(name):
    g = graph(name)
    assert g.row_ptr[-1] == len(g.col) and np.all(np.isin(np.abs(np.log2(g.val)), np.arange(1, 7)))
    if g.n > 1000:
        for L in SHORT + LONG + (HUB,):
            assert np.any(g.lengths == L), L
        assert len(g.long) > 64                           # a second long-row finalize CTA in every solver
        assert np.any(g.col == np.repeat(np.arange(g.n), g.lengths))      # self-loops
        # 64-row blocks that mix long and short rows: row_order is not the identity there
        mixed = [b for b in range(0, g.n, 64) if g.lengths[b:b + 64].max() > 256 and g.lengths[b:b + 64].min() < 10]
        assert len(mixed) > 10
        kinds = {p for (r, p, _) in g.probes if g.lengths[r] > 256}
        assert {0, 255, 256} <= kinds
        # the few-hot columns of the fp16 test reach the hub, the 511 / 512 / 513 rows, long rows of the second
        # finalize CTA and every short length through a planted position
        hit = np.nonzero((g.P @ fewhot_reset(g, 70, 70) != 0).any(axis=1))[0]
        assert {HUB, 511, 512, 513, 255, 256, 1, 2, 3, 5, 7, 9} <= set(g.lengths[hit].tolist())
        assert np.isin(g.long[64:], hit).sum() >= 3
    for B in (37, 64):                                     # the fp32 solver: 1, 2, 3 sweeps
        for iters in (1, 2, 3):
            want = fp32_power_expected(g, dense_reset(g, B, B), iters)
            assert np.all(np.isfinite(want))
    for B in (17, 32, 33, 70):                             # the fp16 solver at (1, 1)
        mixed_11_expected(g, fewhot_reset(g, B, B))
    # the checks themselves: a sum that needs 25 bits, and an fp16 value with 12 significant bits, are refused
    with pytest.raises(AssertionError):
        _fits(np.array([2.0 ** 24]), np.array([0]), 24, "25 bits")
    with pytest.raises(AssertionError):
        assert_fp16(np.array([2049.0]), "12 bits")
    with pytest.raises(AssertionError):
        assert_fp16(np.array([65536.0]), "clamped")


# ------------------------------------------------------------------------------ Chebyshev emulations (w != 1)
def cheb_weights(m):
    """w of sweeps 2..m as the host computes them (double recurrence), then (float)w as the kernels receive it."""
    rho2, w, out = ALPHA * ALPHA, 1.0, []
    for it in range(2, m + 1):
        w = 1.0 / (1.0 - rho2 / 2.0) if it == 2 else 1.0 / (1.0 - rho2 * w / 4.0)
        out.append(float(np.float32(w)))
    return out


def cheb_emulate(g, rhs, x_first, m, ws, store=lambda y: y, prev_of=None):
    """The truncated recurrence of dev_ppr / mixed_cheb: x1 = aP x_first + rhs; x_k = w_k (aP x_{k-1} + rhs) + (1 - w_k)
    x_{k-2} with x_0 = x_first.  Also returns the same recurrence on magnitudes (|w|, |1 - w|), which bounds every
    intermediate sum; `prev_of` replaces the prev buffer (tests of the tolerance itself)."""
    xs, ms = [x_first], [np.abs(x_first)]
    x = store(ALPHA * (g.P @ x_first) + rhs)
    xs.append(x)
    ms.append(ALPHA * (np.abs(g.P) @ ms[0]) + np.abs(rhs))
    for k in range(2, m + 1):
        w = ws[k - 2]
        w1 = float(np.float32(1.0 - w))
        p = xs[k - 2] if prev_of is None else xs[prev_of(k)]
        xs.append(store(w * (ALPHA * (g.P @ xs[k - 1]) + rhs) + w1 * p))
        ms.append(abs(w) * (ALPHA * (np.abs(g.P) @ ms[k - 1]) + np.abs(rhs)) + abs(w1) * ms[k - 2])
    return xs[-1], ms


def _h(x):
    return x.astype(np.float16).astype(np.float64)


def fp32_cheb_expected(g, V, iters, ws=None, prev_of=None):
    """(scores [B, N] float64, per-entry tolerance).  fp32 storage, u = 2^-24: a row of L non-zeros summed in any order
    errs by <= (L + 3) u times its magnitude bound M (the same recurrence on |P|, |v|, |w|, |1 - w|); errors carried in
    from earlier sweeps are bounded by the magnitudes as well, so the error of sweep k is <= k (L_max + 3) u M_k.  The
    normalisation adds 2 u of the result and the bound on the column sum."""
    ws = cheb_weights(iters) if ws is None else ws
    z, ms = cheb_emulate(g, V, V, iters, ws, prev_of=prev_of)
    L = float(max(g.lengths.max(), 1))
    err = iters * (L + 3) * 2.0 ** -24 * ms[-1]
    s = z.sum(axis=0)
    pi = z / s
    tol = err / s + pi * (err.sum(axis=0) / s + 2.0 ** -22)
    return pi.T, tol.T


def mixed_cheb_expected(g, V, m1, m2, ws1=None, ws2=None, prev_of=None):
    """Float64 emulation of the mixed solve with fp16 rounding of every stored iterate (tests/test_mixed_solver_model.py)
    and fp32 w: returns (scores [B, N], tolerance).  Disagreement comes from the fp32 sums ahead of each fp16 rounding:
    they can move a stored value by one fp16 ulp (2^-10 relative).  Through the refinement round, an error e of the
    stored x0 reaches the result only as the residual polynomial of the m2 correction sweeps applied to e (|.| <= the
    magnitude recurrence), so the tolerance is 2^-10 times the magnitudes of every stored iterate, summed over the
    stores, plus the normalisation."""
    ws1 = cheb_weights(m1) if ws1 is None else ws1
    ws2 = cheb_weights(m2) if ws2 is None else ws2
    B = V.shape[1]
    s = column_scale(V.sum(axis=0))
    sv = _h(V * s)
    x0, m_x = cheb_emulate(g, sv, sv, m1, ws1, store=_h, prev_of=prev_of)
    r = _h(T * (ALPHA * (g.P @ x0) + (sv - x0)))
    d, m_d = cheb_emulate(g, r, r, m2, ws2, store=_h, prev_of=prev_of)
    z = x0 + d / T
    u = 2.0 ** -10
    err = u * (sum(m_x[1:]) + np.abs(x0) + np.abs(r) / T + sum(m_d[1:]) / T)
    tot = z.sum(axis=0)
    pi = z / tot
    tol = err / tot + pi * (err.sum(axis=0) / tot + 2.0 ** -22)
    assert np.abs(x0).max() < 65504 and np.abs(r).max() < 65504 and np.abs(d).max() < 65504
    return pi[:, :B].T, tol[:, :B].T


def assert_per_entry(got, want, tol, what, floor=1e-3):
    """|got - want| <= tol on every entry above floor x its column's maximum (relative to the entry, not the max)."""
    big = want >= floor * want.max(axis=1, keepdims=True)
    err = np.abs(got.astype(np.float64) - want)
    bad = big & (err > tol)
    assert not bad.any(), (f"{what}: {np.count_nonzero(bad)} entries off; worst relative error "
                           f"{(err[big] / want[big]).max():.3g} vs tolerance {(tol[big] / want[big]).min():.3g}")
    return big


def _wrong_variants(m):
    """Result-only mistakes a Chebyshev sweep could make: w_k used for w_{k+1}, the w_2 of a / 4, the wrong prev."""
    ws = cheb_weights(m)
    out = []
    if m >= 2:
        out.append(("w_k for w_{k+1}", dict(ws=[1.0] + ws[:-1])))
        out.append(("w_2 with a^2/4", dict(ws=[float(np.float32(1 / (1 - ALPHA ** 2 / 4)))] + ws[1:])))
    if m >= 3:
        out.append(("prev = x_{k-1}", dict(prev_of=lambda k: k - 1)))
    return out


@pytest.mark.parametrize("iters", [2, 3, 5])
def test_fp32_cheb_tolerance_rejects_wrong_recurrences(iters):
    """The per-entry tolerance of the fp32 Chebyshev test is tight enough to fail each wrong recurrence."""
    g = graph("n4133")
    V = dense_reset(g, 8, 3)
    want, tol = fp32_cheb_expected(g, V, iters)
    for name, kw in _wrong_variants(iters):
        alt, _ = fp32_cheb_expected(g, V, iters, **kw)
        with pytest.raises(AssertionError):
            assert_per_entry(alt, want, tol, name)


@pytest.mark.parametrize("m1,m2", [(2, 1), (3, 2)])
def test_mixed_cheb_tolerance_rejects_wrong_recurrences(m1, m2):
    g = graph("n4133")
    V = dense_reset(g, 32, 4)
    want, tol = mixed_cheb_expected(g, V, m1, m2)
    for name, kw in _wrong_variants(m1):
        ws1 = kw.get("ws")
        alt, _ = mixed_cheb_expected(g, V, m1, m2, ws1=ws1, prev_of=kw.get("prev_of"))
        with pytest.raises(AssertionError):
            assert_per_entry(alt, want, tol, name)


# ------------------------------------------------------------------------------ GPU: sweeps against float64
@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def load(hb, g):
    e = hb.Engine(0)
    e.load_graph_csr(g.n, g.row_ptr, g.col, g.val)
    return e


def assert_same(got, want, what):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    bad = got != want
    if bad.any():
        b, n = np.argwhere(bad)[0]
        raise AssertionError(f"{what}: {np.count_nonzero(bad)} entries differ, {np.count_nonzero(bad.any(axis=1))} "
                             f"columns; first column {b} vertex {n}: got {got[b, n]!r}, want {want[b, n]!r}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_fp32_power_sweeps_exact(hb, name):
    """K1 (k_sweep_rows, k_sweep_long_*) at every batch width, 1..3 power sweeps, ragged last sub-batches."""
    g = graph(name)
    e = load(hb, g)
    for width in FP32_WIDTHS:
        e.set_options(ppr_method=hb.PPR_POWER, ppr_precision=hb.PPR_FP32, ppr_batch=width)
        for B in sorted({width, 37 if width == 16 else width + 3}):
            V = dense_reset(g, B, width + B)
            for iters in (1, 2, 3):
                got = e.ppr(V.T.astype(np.float32), iters=iters)
                assert_same(got, fp32_power_expected(g, V, iters), f"{name} width={width} B={B} iters={iters}")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GRAPHS))
def test_mixed_11_exact(hb, name):
    """K1m at mixed_sweeps (1, 1), tol 0: k_sweep_h<false,0,*>, <false,1,true>, the long-row segment / finalize
    kernels, row_order, mixed_prepare_rhs and k_state_to_scores_mixed, bit for bit."""
    g = graph(name)
    e = load(hb, g)
    e.set_options(ppr_precision=hb.PPR_MIXED)
    for B in (17, 32, 33, 70):
        V = fewhot_reset(g, B, B)
        e.reset_stats()
        got = e.ppr(V.T.astype(np.float32), iters=1)
        st = e.stats()
        assert st["ppr_columns"] == 32 * st["ppr_sweeps"] and st["ppr_sweeps"] == 3 * ((B + 31) // 32)
        assert_same(got, mixed_11_expected(g, V), f"{name} B={B}")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("iters", [2, 3, 5])
def test_fp32_chebyshev_epilogue(hb, iters):
    g = graph("n4133")
    e = load(hb, g)
    e.set_options(ppr_method=hb.PPR_CHEBYSHEV, ppr_precision=hb.PPR_FP32)
    for width, B in ((8, 8), (16, 13), (64, 64)):
        e.set_options(ppr_batch=width)
        V = dense_reset(g, B, iters + B)
        want, tol = fp32_cheb_expected(g, V, iters)
        got = e.ppr(V.T.astype(np.float32), iters=iters)
        assert_per_entry(got, want, tol, f"fp32 Chebyshev iters={iters} width={width}")
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("m1,m2", [(2, 1), (3, 2)])
def test_mixed_chebyshev_epilogue(hb, m1, m2):
    g = graph("n4133")
    e = load(hb, g)
    e.set_options(ppr_precision=hb.PPR_MIXED)
    V = dense_reset(g, 40, m1)
    got = e.ppr(V.T.astype(np.float32), iters=m1)         # iters pins (m1, m1 - 1)
    want = np.empty_like(got, np.float64)
    tol = np.empty_like(want)
    for q0 in (0, 32):
        want[q0:q0 + 32], tol[q0:q0 + 32] = mixed_cheb_expected(g, V[:, q0:q0 + 32], m1, m2)
    assert_per_entry(got, want, tol, f"mixed Chebyshev ({m1}, {m2})")
    e.close()


# ------------------------------------------------------------------------------ fp16 saturation at pinned counts
def _saturating_case():
    """Two vertices, P = [[1/2, 1/2], [1/2, 1/2]] (self-loops), reset e_0: s = 16384, x0 = (20480, 4096) and the
    exact residual of the (1, 1) solve is 64 (aP)^2 s e_0 = (131072, 131072) -- twice fp16's 65504."""
    row_ptr = np.array([0, 2, 4], np.int64)
    col = np.array([0, 1, 0, 1], np.int32)
    val = np.full(4, 0.5, np.float32)
    return row_ptr, col, val


def test_saturating_case_on_host():
    import scipy.sparse as sp
    row_ptr, col, val = _saturating_case()
    P = sp.csr_matrix((val.astype(np.float64), col, row_ptr), shape=(2, 2))
    sv = np.array([16384.0, 0.0])
    assert column_scale([1.0])[0] == 16384
    x0 = ALPHA * (P @ sv) + sv
    r = T * (sv - x0 + ALPHA * (P @ x0))
    assert x0.tolist() == [20480.0, 4096.0] and r.tolist() == [131072.0, 131072.0]


@pytest.mark.gpu
def test_mixed_fp16_overflow_is_reported(hb):
    """The pinned (1, 1) solve of the case above would store a residual of 131072, which fp16 cannot hold (sat_h would
    clamp it to 65504 and the answer would be silently wrong): the call must fail instead, also when it is replayed
    from its captured CUDA graph.  The flag is cleared with the error, and at the derived sweep counts the same
    problem is solved correctly on the same handle."""
    row_ptr, col, val = _saturating_case()
    e = hb.Engine(0)
    e.load_graph_csr(2, row_ptr, col, val)
    e.set_options(ppr_precision=hb.PPR_MIXED)
    R = np.zeros((17, 2), np.float32)
    R[:, 0] = 1
    for _ in range(2):
        with pytest.raises(hb.HragError, match="fp16"):
            e.ppr(R, iters=1)
    e.reset_stats()
    out = e.ppr(R)
    assert e.stats()["ppr_columns"] == 32 * e.stats()["ppr_sweeps"]          # the mixed solver ran
    P = np.full((2, 2), 0.5)
    x = np.linalg.solve(np.eye(2) - ALPHA * P, np.array([1.0, 0.0]))
    np.testing.assert_allclose(out, np.tile(x / x.sum(), (17, 1)), rtol=1e-6, atol=0)
    e.close()


@pytest.mark.gpu
def test_unchecked_pinned_solve_does_not_fail_the_next_checked_call(hb, sb):
    """A pinned (1, 1) mixed solve with tol 0 is not checked, but its residual (about a^2 of the rhs) used to stay in
    the running maximum that the next checked call reads, which then failed although its own solve converged.  The
    second pinned call replays the captured CUDA graph of the first (same plan, same buffers): the maximum must be
    cleared after a replay as well."""
    Qi, kept, ks = sb.queries(40, 5)
    R = sb.reset(Qi, kept, ks)
    first = sb.e.ppr(R, iters=1)
    assert_same(sb.e.ppr(R, iters=1), first, "replayed pinned solve")
    sb.e.ppr(R)
    assert 0 < sb.e.stats()["ppr_residual"] < 5e-3
    sb.e.ppr(R, iters=1)
    stage_b = sb.stage_b(Qi, kept, ks, iters=1)           # the pinned compact path, replayed, then a checked call
    sb.stage_b(Qi, kept, ks, iters=1)
    assert_same(sb.stage_b(Qi, kept, ks, iters=1), stage_b, "replayed pinned stage B")
    sb.stage_b(Qi, kept, ks)
    assert 0 < sb.e.stats()["ppr_residual"] < 5e-3


# ------------------------------------------------------------------------------ stage B: compact rhs vs the dense path
class StageB:
    """A synthetic index whose stage-B reset vector is exact on the host: passage embeddings and queries of small
    integers / 4 (the DPR min-max is reproduced by minmax32), passage_node_weight 0.5, kept-fact scores j / 8,
    ent_chunk_count powers of two, link_top_k above the number of phrases (no cut, so no tie at it)."""

    def __init__(self, hb, seed=0):
        from hipporag_b200 import synth
        kg = synth.make_kg(3000, 24_000, seed=seed)
        self.kg = kg
        rng = np.random.default_rng(seed)
        self.P = kg.n_pass
        self.passage_vid = np.asarray(kg.passage_vid, np.int32)
        n = kg.n_nodes
        F = 48
        ents = np.setdiff1d(np.arange(n), self.passage_vid)
        subj = rng.choice(ents, F).astype(np.int32)
        obj = rng.choice(ents, F).astype(np.int32)
        subj[5] = self.passage_vid[7]                         # a phrase seed that is also a passage vertex
        obj[9] = subj[9]                                      # subject == object
        self.cc = (2 ** rng.integers(0, 3, n)).astype(np.int32)
        self.subj, self.obj, self.F = subj, obj, F
        self.Ep = rng.integers(-3, 4, (self.P, 8))
        self.e = hb.Engine(0)
        self.e.load_graph(n, kg.edge_src, kg.edge_dst, kg.edge_w)
        self.e.load_tables(self.passage_vid, subj, obj, self.cc)
        self.e.load_embeddings(np.ones((F, 8), np.float32), (self.Ep / 4).astype(np.float32))

    def queries(self, B, seed):
        rng = np.random.default_rng(seed)
        Qi = rng.integers(-3, 4, (B, 8))
        kept = np.stack([rng.choice(self.F, 5, replace=False) for _ in range(B)]).astype(np.int32)
        ks = (rng.integers(1, 9, (B, 5)) / 8).astype(np.float32)
        kept[0, 0] = 5                                        # the passage-vertex seed
        return Qi, kept, ks

    def reset(self, Qi, kept, ks):
        """float32 reset vectors exactly as k_rhs_passages + k_rhs_seeds (and k_seed_passages + k_seed_scatter) form them."""
        raw = ((Qi @ self.Ep.T).astype(np.float32) / np.float32(16))
        mn = raw.min(axis=1, keepdims=True)
        rg = raw.max(axis=1, keepdims=True) - mn
        with np.errstate(invalid="ignore", divide="ignore"):
            nrm = ((raw - mn) / rg).astype(np.float32)
        nrm[np.broadcast_to(rg == 0, nrm.shape)] = 1
        R = np.zeros((len(Qi), self.kg.n_nodes), np.float32)
        R[:, self.passage_vid] = nrm * np.float32(0.5)
        for q in range(len(Qi)):
            w, occ = {}, {}
            for f, fs in zip(kept[q], ks[q]):
                for v in (int(self.subj[f]), int(self.obj[f])):
                    w[v] = w.get(v, 0.0) + float(np.float32(fs) / np.float32(self.cc[v]))
                    occ[v] = occ.get(v, 0) + 1
            for v in w:
                R[q, v] = R[q, v] + np.float32(w[v] / occ[v])
        return R

    def stage_b(self, Qi, kept, ks, iters=0):
        ids, sc = self.e.stage_b((Qi / 4).astype(np.float32), kept, ks, passage_node_weight=0.5, link_top_k=10,
                                 topk=self.P, iters=iters)
        out = np.zeros((len(Qi), self.P), np.float32)
        np.put_along_axis(out, ids.astype(np.int64), sc, axis=1)
        assert np.all(np.sort(ids, axis=1) == np.arange(self.P))
        return out


@pytest.fixture(scope="module")
def sb(hb):
    s = StageB(hb)
    yield s
    s.e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("B,iters", [(40, 1), (40, 0), (133, 1), (133, 0), (13, 1), (13, 0)])
def test_stage_b_equals_dense_ppr(hb, sb, B, iters):
    """Stage B's passage scores equal hrag_ppr(reset)[:, passage_vid] bit for bit: k_rhs_passages (P = 1000, not a
    multiple of 32; nb < 32 on the last sub-batch), k_rhs_seeds, k_rhs_convert (the x0 scatter) and the passage gathers
    against the dense path, for the mixed solver (B > 16; 133 = five sub-batches, both buffer sets reused) and the fp32
    solver (B <= 16)."""
    assert sb.P % 32 != 0
    Qi, kept, ks = sb.queries(B, B + iters)
    sb.e.reset_stats()
    got = sb.stage_b(Qi, kept, ks, iters)
    st = sb.e.stats()
    assert (st["ppr_columns"] == 32 * st["ppr_sweeps"]) == (B > 16)
    R = sb.reset(Qi, kept, ks)
    want = sb.e.ppr(R, iters=iters)[:, sb.passage_vid]
    assert_same(got, want, f"stage B vs hrag_ppr B={B} iters={iters}")


def _permutations(B, rng):
    return {"reversed": np.arange(B)[::-1], "rotated": np.roll(np.arange(B), 31), "shuffled": rng.permutation(B)}


@pytest.mark.gpu
def test_stage_b_column_and_batch_invariance(hb, sb):
    """Every column of a sweep is computed on its own, so a query's scores do not depend on its column (0 .. 31), on its
    sub-batch (buffer set 0 or 1, a first or a replayed CUDA graph) or on its neighbours.  k_rhs_seeds adds the seed
    weights into vsum with a double atomicAdd in no fixed order; vsum only sets the power-of-two column scale
    (2^floor(log2(16384 / vsum))), and on these inputs it is at least 0.5 x 1000 passages x the mean min-max score away
    from any power-of-two boundary by far more than the few units of 2^-40 that reordering double additions of float32
    weights can move it, so the scale cannot change."""
    rng = np.random.default_rng(1)
    B = 133
    Qi, kept, ks = sb.queries(B, 99)
    kept[40:48] = kept[39]                                # queries sharing every seed vertex: the atomicCAS path
    ks[40:48] = ks[39]
    base = sb.stage_b(Qi, kept, ks)
    for name, perm in _permutations(B, rng).items():
        got = sb.stage_b(Qi[perm], kept[perm], ks[perm])
        assert_same(got, base[perm], f"stage B, {name} queries")
    for q in (0, 39, 132):                                # one query in all 32 columns
        same = np.full(32, q)
        got = sb.stage_b(Qi[same], kept[same], ks[same])
        assert_same(got, np.repeat(base[q:q + 1], 32, axis=0), f"stage B, query {q} in every column")
    vs = sb.reset(Qi, kept, ks).astype(np.float64).sum(axis=1)
    frac = np.log2(16384 / vs) - np.floor(np.log2(16384 / vs))
    assert np.all((frac > 1e-6) & (frac < 1 - 1e-6))       # no column sum near a power of two


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "mixed"])
def test_dense_ppr_column_invariance(hb, sb, precision):
    rng = np.random.default_rng(2)
    B = 133 if precision == "mixed" else 16
    Qi, kept, ks = sb.queries(B, 7)
    R = sb.reset(Qi, kept, ks)
    e = sb.e
    e.set_options(ppr_precision=hb.PPR_MIXED)
    if precision == "fp32":
        e.set_options(ppr_batch=16)
    try:
        base = e.ppr(R)
        for name, perm in _permutations(B, rng).items():
            assert_same(e.ppr(R[perm]), base[perm], f"hrag_ppr {precision}, {name}")
        rep = np.repeat(R[3:4], 32 if precision == "mixed" else 16, axis=0)
        assert_same(e.ppr(rep), np.repeat(base[3:4], len(rep), axis=0), f"hrag_ppr {precision}, one vector everywhere")
    finally:
        e.set_options(ppr_batch=16)
