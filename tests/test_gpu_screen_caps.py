"""The stage-A screen at and past each of its caps, against a numpy model of its accounting and the float64 oracle.

The screen (DESIGN.md section 4, K2) lists candidates per query from the hi.hi tile lists (k_screen_select), stages
them per 128-query m-tile (k_screen_stage), rescores the staged tiles with the split product and selects over them
(k_screen_finish).  It claims the exact outputs, or a raised flag and a counted fallback, and that claim rests on three
caps (kernels.h): 256 listed candidates and 8 saturated tiles per query, 48 staged tiles per m-tile.  screen_model()
below is that accounting written down once, from exact s1 = q_hi.e_hi, s4 = the split product and the bound E_q:

  per query    L (the 8th best s1), U (the smallest s1), the bands s1 >= L - 2 E_q and s1 <= U + 2 E_q; per 256-row
               tile min(8, in-band keys) listed plus the tile's two smallest rows where they are in band; a tile is
               saturated when it has 8 keys in the upper band or its second smallest row is in the lower band;
  per m-tile   the distinct staged rows (the candidates and every row f < F of each saturated tile), counted per
               column f mod 256;
  per chunk    (1,024 queries) a fallback when a query lists more than 256 candidates or 8 saturated tiles, an m-tile
               has a column with more than 48 staged rows, or E_q is not finite;
  per call     the fallbacks, and the lo rows the gather reads: per m-tile and column min(count, 48) (exact when no
               query overflows its own caps: the staging claims a column's first 48 rows in any order).

Where no chunk falls back it also gives the screen's outputs: the selection over the m-tile's staged rows.  The inputs
are family A of test_gpu_split_exact (small-integer hi parts, lo = c 2^-12, queries without lo), exact in fp32, with
groups of queries that share a sign pattern and rows planted at the group's top and bottom s1 levels, one hi row each,
so lo decides within every tie.  The CPU tests check each case's premises and that every cap one lower or higher, a
band of E_q, the second-smallest rule dropped, staging shared across m-tiles or per query, and saturated tiles that
stage only their listed rows would each change a predicted fallback count or an expected output.  The GPU tests run
every case at two CTA counts on resident planes and with the lo plane on the host, against the float64 oracle bit for
bit, with the fallback count and the gathered lo bytes the model predicts.
"""
import functools

import numpy as np
import pytest

from tests.test_gpu_selection_exact import assert_same, expected_topk, minmax32, ranking
from tests.test_gpu_split_exact import LO_A, _err_bound64, _stored, exact_scores

CAND_CAP, SAT_CAP, STAGE_CAP = 256, 8, 48   # kScreenCandidates, kScreenSatTiles, kScreenStageTiles (kernels.h)
CHUNK, MTILE, TILE = 1024, 128, 256         # queries per screened chunk, per m-tile; facts per tile
F = 65_536 + 37                             # screened; 257 tiles, the last one ragged (37 rows)
D = 72                                      # a multiple of 8, not of 16, 32 or 64
N_TILES = -(-F // TILE)
COL = 77                                    # the column f mod 256 the staged-tile cases fill


# ------------------------------------------------------------------------------ the model
RULES = dict(cand_cap=CAND_CAP, sat_cap=SAT_CAP, stage_cap=STAGE_CAP, band=2.0, second_low=True, staging="m-tile",
             whole_tile=True)


def screen_bound(qh, ql, eh, el):
    """E_q as k_query_err computes it, in float64 with its (1 + 2^-10) factor."""
    return _err_bound64(qh, ql, eh, el) * (1 + 2.0 ** -10)


def query_accounting(s1, E, rules=RULES):
    """k_screen_select for one query row s1 [F]: n (the kernel's pushes: a row both listed and low counts twice),
    the candidate rows, the saturated tiles, L and U."""
    if not np.isfinite(E):
        return dict(n=0, rows=np.zeros(0, np.int64), sat=[], bad=True, L=np.nan, U=np.nan)
    L = np.partition(s1, s1.size - 8)[s1.size - 8] if s1.size >= 8 else -np.inf
    U = s1.min()
    up = np.flatnonzero(s1 >= L - rules["band"] * E)
    low = np.flatnonzero(s1 <= U + rules["band"] * E)
    pushed, sat = [], set()
    for t in np.unique(up // TILE):
        r = up[up // TILE == t]
        r = r[np.lexsort((r, -s1[r]))][:8]              # the tile's list: s1 descending, then index ascending
        pushed.extend(r.tolist())
        if r.size == 8:
            sat.add(int(t))
    for t in np.unique(low // TILE):
        r = low[low // TILE == t]
        r = r[np.lexsort((r, s1[r]))][:2]               # the tile's two smallest: s1 ascending, then index
        pushed.extend(r.tolist())
        if r.size == 2 and rules["second_low"]:
            sat.add(int(t))
    return dict(n=len(pushed), rows=np.unique(np.asarray(pushed, np.int64)), sat=sorted(sat), bad=False, L=L, U=U)


def _staged_rows(acc, rules):
    rows = [acc["rows"]]
    if rules["whole_tile"]:
        for t in acc["sat"][:rules["sat_cap"]]:
            rows.append(np.arange(t * TILE, min(t * TILE + TILE, F)))
    return np.unique(np.concatenate(rows))


def screen_model(s1, s4, E, qidx, rules=RULES):
    """The screen over a call whose query b is unique query qidx[b] (s1 / s4 float32 [n_unique, F], E [n_unique]).
    Returns per-unique-query accounting, per-chunk records (flagged, gathered rows, whether that count is exact, the
    staged pools of its m-tiles) and the call's fallbacks and gathered rows."""
    qidx = np.asarray(qidx)
    acc = [query_accounting(s1[u].astype(np.float64), float(E[u]), rules) for u in range(s1.shape[0])]
    for u, a in enumerate(acc):                         # k_screen_finish's |s4 - s1| <= E_q on the listed rows
        r = a["rows"]
        a["check"] = bool(np.all(np.abs(s4[u, r].astype(np.float64) - s1[u, r]) <= E[u]))
        a["staged"] = _staged_rows(a, rules)
    chunks = []
    for q0 in range(0, qidx.size, CHUNK):
        rows = qidx[q0:q0 + CHUNK]
        us = np.unique(rows)
        over_q = any(acc[u]["bad"] or acc[u]["n"] > rules["cand_cap"] or len(acc[u]["sat"]) > rules["sat_cap"]
                     or not acc[u]["check"] for u in us)
        # "m-tile": the kernel; "chunk": one staging shared by the chunk's m-tiles; "query": per m-tile, without
        # pos_of's dedupe across its queries
        groups = [rows] if rules["staging"] == "chunk" else [rows[i:i + MTILE] for i in range(0, rows.size, MTILE)]
        pools, over_col, gathered, max_col = [], False, 0, 0
        for g in groups:
            if rules["staging"] == "query":
                counts = sum(np.bincount(acc[u]["staged"] % TILE, minlength=TILE) for u in g)
                pool = np.unique(np.concatenate([acc[u]["staged"] for u in g]))
            else:
                pool = np.unique(np.concatenate([acc[u]["staged"] for u in np.unique(g)]))
                counts = np.bincount(pool % TILE, minlength=TILE)
            max_col = max(max_col, int(counts.max()))
            over_col |= bool(counts.max() > rules["stage_cap"])
            gathered += int(np.minimum(counts, rules["stage_cap"]).sum())
            pools.append((g, pool))
        chunks.append(dict(q0=q0, nb=rows.size, flagged=over_q or over_col, gathered=gathered, exact=not over_q,
                           max_col=max_col, pools=pools))
    return dict(acc=acc, chunks=chunks, fallbacks=sum(c["flagged"] for c in chunks),
                gathered=sum(c["gathered"] for c in chunks))


def _select(s, rows):
    """(8 best ids, their s4, min, max) of one query's scores s over `rows` (ids ascending breaks ties)."""
    v = s[rows]
    o = np.lexsort((rows, -v))[:8]
    return rows[o], v[o], v.min(), v.max()


def model_outputs(model, s4, qidx):
    """What the screen returns for each call row: the selection over its m-tile's staged rows, or over all facts
    where its chunk falls back (the exact path).  [B, 8] ids and raw s4, [B, 2] (min, max)."""
    B = np.asarray(qidx).size
    ids, sc, mm = np.zeros((B, 8), np.int64), np.zeros((B, 8), np.float32), np.zeros((B, 2), np.float32)
    everything = np.arange(F)
    exact = {}
    for c in model["chunks"]:
        b = c["q0"]
        for g, pool in c["pools"]:                      # consecutive call rows
            memo = {}
            for j, u in enumerate(g):
                if u not in memo:
                    if c["flagged"]:
                        if u not in exact:
                            exact[u] = _select(s4[u], everything)
                        memo[u] = exact[u]
                    else:
                        memo[u] = _select(s4[u], pool)
                i, v, lo, hi = memo[u]
                ids[b + j], sc[b + j], mm[b + j] = i, v, (lo, hi)
            b += len(g)
    return ids, sc, mm


# ------------------------------------------------------------------------------ the inputs
class World:
    """F family-A fact rows: fillers with hi +-1/4 and lo in {-1, 0, 1} 2^-12, and rows planted for groups of
    queries.  Group g has a sign pattern sigma_g; its queries are sigma_g m / 4 with m = 1 on column 0 and on 35 of
    the other columns, 2 on the remaining 36 (so every query of every group has the same norm and the same sum of m,
    108).  A row planted at level +1 (-1) has hi +2 sigma_g / 4 (-2 sigma_g / 4): s1 = +-13.5 for every query of the
    group, far from the fillers (s1 within about +-4) and from other groups' rows (about +-8).  `shift` moves column 0
    one step toward zero, which moves s1 by 1/16 toward zero.  Its lo is t sigma_g 2^-12 (t per row: s4 - s1 =
    t 108 2^-14 for the whole group) or random in -3..3 (the order then differs from query to query); |c| <= 1 on a
    shifted column 0, whose hi is +-1/4."""

    def __init__(self, seed, n_groups):
        self.rng = np.random.default_rng([seed, 7])
        self.sigma = self.rng.choice([-1, 1], (n_groups, D))
        self.a = self.rng.choice([-1, 1], (F, D))
        self.c = self.rng.integers(-1, 2, (F, D))
        self.used = np.zeros(F, bool)
        self.tops = [[] for _ in range(n_groups)]       # the rows of each group's s1 levels (for the premises)
        self.bottoms = [[] for _ in range(n_groups)]
        self.near = [[] for _ in range(n_groups)]       # rows one 1/16 step inside a level
        self.queries = {}

    def plant(self, g, rows, level, t=None, shift=0):
        rows = np.atleast_1d(np.asarray(rows, np.int64))
        assert rows.max() < F and not self.used[rows].any() and np.unique(rows).size == rows.size
        self.used[rows] = True
        s = self.sigma[g]
        a = np.tile(2 * level * s, (rows.size, 1))
        a[:, 0] -= shift * level * s[0]
        if t is None:
            c = self.rng.integers(-3, 4, (rows.size, D))
        else:
            c = np.outer(np.broadcast_to(t, rows.shape), s)
        if shift:
            c[:, 0] = np.clip(c[:, 0], -1, 1)
        self.a[rows], self.c[rows] = a, c
        (self.near if shift else self.tops if level > 0 else self.bottoms)[g].extend(rows.tolist())
        return rows

    def tile_rows(self, tile, n, avoid=()):
        """n distinct free rows of a tile, at random columns (not in `avoid`), ascending."""
        r = np.arange(tile * TILE, min(tile * TILE + TILE, F))
        r = r[~self.used[r] & ~np.isin(r % TILE, avoid)]
        return np.sort(self.rng.choice(r, n, replace=False))

    def group_queries(self, g, n):
        m = np.ones((n, D), np.int64)
        for i in range(n):
            m[i, 1 + self.rng.choice(D - 1, 36, replace=False)] = 2
        q = self.sigma[g] * m
        self.queries[g] = q
        return q

    def finish(self, calls):
        """calls: name -> [(group, query numbers)], the call's rows in order.  Scores, bounds and each call's unique
        query index."""
        groups = sorted(self.queries)
        base = np.cumsum([0] + [self.queries[g].shape[0] for g in groups])
        first = dict(zip(groups, base))
        qh = np.concatenate([self.queries[g] for g in groups]) / 4.0
        ql = np.zeros_like(qh)
        eh, el = self.a / 4.0, self.c * LO_A
        w = dict(Q=_stored(qh, ql), E=_stored(eh, el), qh=qh, ql=ql, eh=eh, el=el, tops=self.tops,
                 bottoms=self.bottoms, near=self.near, group_of=np.repeat(groups, np.diff(base)))
        w["s4"], w["s1"] = exact_scores(qh, ql, eh, el)
        w["Eq"] = screen_bound(qh, ql, eh, el)
        w["calls"] = {name: np.concatenate([first[g] + np.asarray(ix) for g, ix in parts])
                      for name, parts in calls.items()}
        return w


def _spread(world, g, tiles, per_tile, n, **kw):
    """n rows of group g at level +1, per_tile in each of `tiles` (fewer in the last one used)."""
    out = []
    for t in tiles:
        k = min(per_tile, n - len(out))
        if k <= 0:
            break
        out.extend(world.plant(g, world.tile_rows(t, k), +1, **kw).tolist())
    assert len(out) == n
    return out


@functools.lru_cache(maxsize=None)
def world_candidates():
    """Case a.  Group 0 (127 queries, 67 more for the multi-chunk call) and group 1 (1 query) each have 255 rows tied
    at the top, at most 7 per tile, and one bottom row: 256 listed candidates per query, no tile saturated.  Group 2
    (1 query) has 256 tied rows: 257 candidates."""
    w = World(1, 3)
    for g, (t0, n) in enumerate(((0, 255), (40, 255), (80, 256))):
        _spread(w, g, range(t0, t0 + 37), 7, n)
        w.plant(g, w.tile_rows(120 + g, 1), -1)
    w.group_queries(0, 127 + 67)
    w.group_queries(1, 1)
    w.group_queries(2, 1)
    at = [(1, [0]), (0, range(127))]
    over = [(2, [0]), (0, range(127))]
    tail = [(1, [0]), (0, range(127, 127 + 67))]           # 68 queries: a ragged m-tile
    calls = {"candidates at cap": at, "candidates past cap": over,
             "three chunks, one past cap": at * 8 + at * 7 + over + at * 3 + tail,
             "three chunks at cap": at * 8 + at * 8 + at * 3 + tail}
    return w.finish(calls)


def _saturate_upper(w, g, tile, rows=None):
    """16 rows of `tile` tied at the top: the list keeps the 8 lowest, whose lo is against the queries (t -3..-1);
    the 8 others have t 1..7, so the group's true top 8 are unlisted rows of saturated tiles."""
    rows = w.tile_rows(tile, 16) if rows is None else np.asarray(rows)
    w.plant(g, rows[:8], +1, t=w.rng.integers(-3, 0, 8))
    w.plant(g, rows[8:], +1, t=w.rng.integers(1, 8, 8))


def _saturate_lower(w, g, tile, t_min):
    """3 rows of `tile` tied at the bottom: the two low entries are the lowest two (lo t = 3, raising s4); the third,
    with t = t_min, holds the tile's smallest s4."""
    rows = w.tile_rows(tile, 3)
    w.plant(g, rows[:2], -1, t=3)
    w.plant(g, rows[2:], -1, t=t_min)


@functools.lru_cache(maxsize=None)
def world_saturated():
    """Case b.  Group 0: 5 tiles and the ragged last tile saturated from the upper band, 2 tiles from the lower band
    (second smallest in band), 8 in all; its true minimum is the third row of a lower tile.  Group 1: the same with 6
    upper tiles, 9 in all.  Both use the last tile (rows 65,536 .. 65,572)."""
    w = World(2, 2)
    for g, upper, lower in ((0, (10, 20, 30, 40, 50), (60, 70)), (1, (110, 120, 130, 140, 150, 160), (170, 180))):
        for t in upper:
            _saturate_upper(w, g, t)
        _saturate_upper(w, g, N_TILES - 1, rows=np.arange(65_536, 65_552) if g == 0 else np.arange(F - 16, F))
        _saturate_lower(w, g, lower[0], -5)
        _saturate_lower(w, g, lower[1], -4)
        w.group_queries(g, 128)
    return w.finish({"saturated tiles at cap": [(0, range(128))], "saturated tiles past cap": [(1, range(128))]})


def _sizes(n_groups, n=MTILE):
    return [n // n_groups + (i < n % n_groups) for i in range(n_groups)]


@functools.lru_cache(maxsize=None)
def world_staged():
    """Case c, one column.  Groups 0..5 (one m-tile) each have 8 rows tied at the top, all at column COL of 8
    distinct tiles: 48 rows at that column, each in its group's top 8.  Group 6 adds one more such row (and 7 at
    other columns); groups 7..12 put 48 more rows at COL, for the second m-tile of a 256-query call.  Bottom rows sit
    at other columns."""
    w = World(3, 13)
    tile = iter(range(N_TILES - 1))
    for g in range(13):
        n_col = 1 if g == 6 else 8
        for _ in range(n_col):
            w.plant(g, next(tile) * TILE + COL, +1)
        for _ in range(8 - n_col):
            w.plant(g, w.tile_rows(next(tile), 1, avoid=[COL]), +1)
        w.plant(g, w.tile_rows(200 + g, 1, avoid=[COL]), -1)
    for g in range(13):
        w.group_queries(g, 22)
    six, seven = _sizes(6), _sizes(7)
    return w.finish({
        "48 staged rows in a column": [(g, range(n)) for g, n in zip(range(6), six)],
        "49 staged rows in a column": [(g, range(n)) for g, n in zip(range(7), seven)],
        "48 + 48 over two m-tiles": [(g, range(n)) for g, n in zip(range(6), six)]
                                    + [(g, range(n)) for g, n in zip(range(7, 13), six)],
    })


@functools.lru_cache(maxsize=None)
def world_filled():
    """Case c, every column.  Groups 0..5 each saturate 8 tiles (8 rows tied at the top in each), 48 tiles in one
    m-tile: every column holds 48 staged rows; each group's bottom row lies in one of its own saturated tiles.  Group 6
    takes group 0's place with 8 other tiles and its bottom row outside every saturated tile: one more candidate."""
    w = World(4, 7)
    for g in range(7):
        tiles = range(8 * g, 8 * g + 8)
        for t in tiles:
            w.plant(g, w.tile_rows(t, 8), +1)
        w.plant(g, w.tile_rows(100 if g == 6 else tiles[0], 1), -1)
        w.group_queries(g, 22)
    six = _sizes(6)
    return w.finish({"48 saturated tiles in an m-tile": [(g, range(n)) for g, n in zip(range(6), six)],
                     "48 saturated tiles and one more row": [(g, range(n)) for g, n in zip((6, 1, 2, 3, 4, 5), six)]})


@functools.lru_cache(maxsize=None)
def world_band():
    """Case d.  8 rows tied at the top (4 with lo t = -3 against the queries), one row 1/16 below them with t = 7: it
    is fifth in s4, and its s1 lies between L - 2 E_q and L - E_q.  Two rows tied at the bottom with t = 3 and one row
    1/16 above them with t = -7, which holds the s4 minimum from between U + E_q and U + 2 E_q.  The rows with |t| = 7
    set the largest lo norm, which puts E_q near 0.049: 1/16 is 1.28 E_q."""
    w = World(5, 1)
    t = np.array([-3, -3, -3, -3, -2, 0, 1, 3])
    w.rng.shuffle(t)
    for i, ti in enumerate(t):
        w.plant(0, w.tile_rows(5 + i, 1), +1, t=ti)
    w.plant(0, w.tile_rows(20, 1), +1, t=7, shift=1)
    for tile in (30, 31):
        w.plant(0, w.tile_rows(tile, 1), -1, t=3)
    w.plant(0, w.tile_rows(40, 1), -1, t=-7, shift=1)
    w.group_queries(0, 128)
    return w.finish({"band rows": [(0, range(128))]})


WORLDS = (world_candidates, world_saturated, world_staged, world_filled, world_band)
# (world, call, designed fallbacks)
CASES = {
    "candidates at cap": (world_candidates, 0),
    "candidates past cap": (world_candidates, 1),
    "saturated tiles at cap": (world_saturated, 0),
    "saturated tiles past cap": (world_saturated, 1),
    "48 staged rows in a column": (world_staged, 0),
    "49 staged rows in a column": (world_staged, 1),
    "48 + 48 over two m-tiles": (world_staged, 0),
    "48 saturated tiles in an m-tile": (world_filled, 0),
    "48 saturated tiles and one more row": (world_filled, 1),
    "band rows": (world_band, 0),
    "three chunks, one past cap": (world_candidates, 1),
    "three chunks at cap": (world_candidates, 0),
}
SINGLE = [n for n in CASES if not n.startswith("three chunks")]


@functools.lru_cache(maxsize=None)
def case_model(name, **rules):
    w = CASES[name][0]()
    return screen_model(w["s1"], w["s4"], w["Eq"], w["calls"][name], dict(RULES, **rules))


# ------------------------------------------------------------------------------ CPU: the model by hand
def test_model_hand_worked():
    """Two queries of one m-tile on hand-set s1 (E_q = 0.1).  Query 0: 9 rows tied at 10 in tile 0 (its list holds
    rows 0..7: saturated), rows 300 and 301 tied at -5 (tile 1: both low entries in band, saturated), row 700 at
    9.85 (in the band L - 0.2), row 701 at 9.75 (not).  Query 1: the same rows, no ties below, 3 rows at 10."""
    s1 = np.zeros((2, F), np.float32)
    s1[0, :9] = 10
    s1[0, [300, 301]] = -5
    s1[0, 700], s1[0, 701] = 9.85, 9.75
    s1[1, [5, 600, 601]] = 10
    s1[1, 1000:1005] = 9.9
    s1[1, 2000] = -3
    E = np.array([0.1, 0.1])
    a0 = query_accounting(s1[0].astype(np.float64), 0.1)
    assert a0["L"] == 10 and a0["U"] == -5
    assert a0["n"] == 8 + 1 + 2 and a0["sat"] == [0, 1]
    assert a0["rows"].tolist() == list(range(8)) + [300, 301, 700]
    a1 = query_accounting(s1[1].astype(np.float64), 0.1)
    assert a1["n"] == 3 + 5 + 1 and a1["sat"] == [] and np.float32(a1["L"]) == np.float32(9.9)
    m = screen_model(s1, s1, E, [0, 1])
    (g, pool), = m["chunks"][0]["pools"]
    # tiles 0 and 1 whole, row 700, and query 1's rows 600, 601, 1000..1004, 2000 (row 5 is in tile 0 already)
    assert pool.tolist() == list(range(512)) + [600, 601, 700] + list(range(1000, 1005)) + [2000]
    assert m["fallbacks"] == 0 and m["gathered"] == pool.size
    assert m["chunks"][0]["max_col"] == 3                  # e.g. column 88: rows 88, 344 and 600
    # a cap of 10 candidates and 1 saturated tile: query 0 overflows both
    assert screen_model(s1, s1, E, [0, 1], dict(RULES, cand_cap=10))["fallbacks"] == 1
    assert screen_model(s1, s1, E, [0, 1], dict(RULES, sat_cap=1))["fallbacks"] == 1
    # 1,100 copies of query 1 and one of query 0: two chunks, the second at rows 1,024..1,100
    m = screen_model(s1, s1, E, [1] * 1030 + [0] * 70, dict(RULES, cand_cap=10))
    assert [c["flagged"] for c in m["chunks"]] == [False, True] and m["fallbacks"] == 1
    # E_q not finite: the chunk falls back
    assert screen_model(s1, s1, np.array([0.1, np.inf]), [0, 1])["fallbacks"] == 1
    # the selection over the staged pool is the exact one
    ids, sc, mm = model_outputs(screen_model(s1, s1, E, [0, 1]), s1, [0, 1])
    assert ids[0].tolist() == list(range(8)) and ids[1].tolist() == [5, 600, 601, 1000, 1001, 1002, 1003, 1004]
    assert mm.tolist() == [[-5, 10], [-3, 10]]


# ------------------------------------------------------------------------------ CPU: the premises of every case
def _reach_bits(w):
    """Bits from the largest partial sum of any dot product (at most sum |q_hi| (|e_hi| + |e_lo|); q_lo = 0) down to
    the 2^-14 quantum of family A's products."""
    reach = np.abs(w["qh"]) @ (np.abs(w["eh"]) + np.abs(w["el"])).T
    return int(np.ceil(np.log2(reach.max() / 2.0 ** -14 + 1)))


@functools.lru_cache(maxsize=None)
def exact_outputs(world):
    w = world()
    s4 = w["s4"]
    order = np.argsort(-s4, axis=1, kind="stable")[:, :8]
    return order, np.take_along_axis(s4, order, 1), np.stack([s4.min(1), s4.max(1)], 1)


# the statistic each case puts exactly at its cap (or one past it)
AT = {
    "candidates at cap": ("candidates", CAND_CAP), "candidates past cap": ("candidates", CAND_CAP + 1),
    "saturated tiles at cap": ("saturated", SAT_CAP), "saturated tiles past cap": ("saturated", SAT_CAP + 1),
    "48 staged rows in a column": ("column", STAGE_CAP), "49 staged rows in a column": ("column", STAGE_CAP + 1),
    "48 + 48 over two m-tiles": ("column", STAGE_CAP), "48 saturated tiles in an m-tile": ("column", STAGE_CAP),
    "48 saturated tiles and one more row": ("column", STAGE_CAP + 1), "three chunks at cap": ("candidates", CAND_CAP),
    "three chunks, one past cap": ("candidates", CAND_CAP + 1),
}


@pytest.mark.parametrize("name", list(CASES))
def test_case_premise(name):
    """The case is exact in fp32 (every partial sum within 22 bits), its planted rows tie at their group's levels
    with lo deciding inside each tie, every s1 level is at least 0.2 E_q from each band edge (L - 2 E_q, L - E_q,
    U + E_q, U + 2 E_q), the statistic of its cap sits where it was designed, the model predicts the designed
    fallbacks, and where no chunk falls back the selection over the staged rows is the exact one."""
    world, designed = CASES[name]
    w = world()
    qidx = w["calls"][name]
    m = case_model(name)
    assert _reach_bits(w) <= 22
    s1, s4, E = w["s1"].astype(np.float64), w["s4"], w["Eq"]
    for u in np.unique(qidx):
        g, a = w["group_of"][u], m["acc"][u]
        top, bottom, near = w["tops"][g], w["bottoms"][g], w["near"][g]
        assert np.all(s1[u, top] == a["L"]) and np.all(s1[u, bottom] == a["U"])
        assert set(np.flatnonzero(s1[u] >= a["L"] - 2 * E[u])) == set(top) | {r for r in near if s1[u, r] > 0}
        assert set(np.flatnonzero(s1[u] <= a["U"] + 2 * E[u])) == set(bottom) | {r for r in near if s1[u, r] < 0}
        for rows in (top, bottom):
            if len(rows) > 2:
                assert np.unique(s4[u, rows]).size > 1
        levels = np.unique(s1[u])
        for edge in (a["L"] - 2 * E[u], a["L"] - E[u], a["U"] + E[u], a["U"] + 2 * E[u]):
            assert np.abs(levels - edge).min() >= 0.2 * E[u], (name, u, edge)
    stat, value = AT.get(name, (None, None))
    us = np.unique(qidx)
    got = {"candidates": max(m["acc"][u]["n"] for u in us), "saturated": max(len(m["acc"][u]["sat"]) for u in us),
           "column": max(c["max_col"] for c in m["chunks"])}
    if stat:
        assert got[stat] == value, (name, got)
    if name in ("candidates at cap", "three chunks at cap"):
        assert all(m["acc"][u]["n"] == CAND_CAP for u in us)             # every query at the cap
    assert got["candidates"] <= CAND_CAP or stat == "candidates"
    assert got["saturated"] <= SAT_CAP or stat == "saturated"
    assert m["fallbacks"] == designed
    ids, sc, mm = model_outputs(m, s4, qidx)
    o_ids, o_sc, o_mm = (x[qidx] for x in exact_outputs(world))
    assert np.array_equal(ids, o_ids) and np.array_equal(sc, o_sc) and np.array_equal(mm, o_mm)


def test_only_staging_finds_the_answer():
    """Case b: the true top 8 are unlisted rows of saturated tiles and the true minimum is no listed candidate; case
    d: the rows inside the bands are in the s4 top 8 and hold the s4 minimum."""
    w = world_saturated()
    m = case_model("saturated tiles at cap")
    order, _, mm = exact_outputs(world_saturated)
    for u in np.unique(w["calls"]["saturated tiles at cap"]):
        listed = set(m["acc"][u]["rows"].tolist())
        assert not set(order[u].tolist()) & listed
        assert np.flatnonzero(w["s4"][u] == mm[u, 0])[0] not in listed
    w = world_band()
    order, _, mm = exact_outputs(world_band)
    up, down = sorted(w["near"][0], key=lambda r: -w["s1"][0, r])
    E = w["Eq"]
    assert np.all(np.abs(E - 0.0487) < 0.001)
    for u in range(w["Q"].shape[0]):
        assert up in order[u].tolist() and w["s4"][u, down] == mm[u, 0]
        assert np.unique(w["s4"][u]).size > 1 and w["s4"][u, down] < w["s4"][u, w["bottoms"][0]].min()


# ------------------------------------------------------------------------------ CPU: each rule matters
MUTATIONS = {
    "candidate cap 255": (dict(cand_cap=CAND_CAP - 1), ["candidates at cap", "three chunks at cap"]),
    "candidate cap 257": (dict(cand_cap=CAND_CAP + 1), ["candidates past cap", "three chunks, one past cap"]),
    "saturated cap 7": (dict(sat_cap=SAT_CAP - 1), ["saturated tiles at cap"]),
    "saturated cap 9": (dict(sat_cap=SAT_CAP + 1), ["saturated tiles past cap"]),
    "stage cap 47": (dict(stage_cap=STAGE_CAP - 1), ["48 staged rows in a column", "48 + 48 over two m-tiles",
                                                     "48 saturated tiles in an m-tile"]),
    "stage cap 49": (dict(stage_cap=STAGE_CAP + 1), ["49 staged rows in a column",
                                                     "48 saturated tiles and one more row"]),
    "bands of E_q": (dict(band=1.0), ["band rows"]),
    "no second-smallest saturation": (dict(second_low=False), ["saturated tiles at cap", "saturated tiles past cap"]),
    "staging shared across m-tiles": (dict(staging="chunk"), ["48 + 48 over two m-tiles"]),
    "staging per query": (dict(staging="query"), ["candidates at cap", "48 saturated tiles in an m-tile"]),
    "saturated tiles stage listed rows only": (dict(whole_tile=False), ["saturated tiles at cap"]),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_mutations_change_the_prediction(mutation):
    """Each variant of the rules changes, on the named cases, the predicted fallback count or the predicted ids,
    scores or (min, max): the GPU tests below, which assert both, would fail on a kernel that followed it."""
    rules, names = MUTATIONS[mutation]
    for name in names:
        world = CASES[name][0]
        w = world()
        qidx = w["calls"][name]
        good, bad = case_model(name), case_model(name, **rules)
        same = good["fallbacks"] == bad["fallbacks"] and all(
            np.array_equal(x, y) for x, y in zip(model_outputs(good, w["s4"], qidx), model_outputs(bad, w["s4"], qidx)))
        assert not same, f"{mutation}: {name} predicts the same"


# ------------------------------------------------------------------------------ GPU: every case, bit for bit
@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def _lo_budget():
    """The hi plane plus two 256-row lo slices."""
    return F * D * 2 + 2 * 256 * D * 2 + 100


def _engine(hb, w, lo_host):
    if lo_host:
        e = hb.Engine(0, fact_device_bytes=_lo_budget(), fact_lo_on_host=True)
    else:
        e = hb.Engine(0)
    e.load_embeddings(w["E"], w["E"][:4])
    assert e.fact_planes_info()["on_host"] == (2 if lo_host else 0)
    return e


@functools.lru_cache(maxsize=None)
def _oracle(world):
    s4 = world()["s4"]
    return minmax32(s4), ranking(s4)[:, :64], np.stack([s4.min(1), s4.max(1)], 1)


def _run(e, world, name, fallbacks, ks=(1, 5, 8)):
    """stage_a of the call at 0 and 7 GEMM CTAs against the float64 oracle: ids, min-max scores, n_valid, the
    per-query (min, max) when the call is one chunk, and the fallback count.  Returns the h2d bytes of each call."""
    w = world()
    qidx = w["calls"][name]
    norm, order, mm = _oracle(world)
    Q = w["Q"][qidx]
    h2d = []
    try:
        for ctas in (0, 7):
            e.debug_sim_ctas(ctas)
            for k in ks:
                e.reset_stats()
                idx, sc, nv = e.stage_a(Q, k)
                st = e.stats()
                want_idx, want_sc, want_nv = expected_topk(norm, order, k)
                tag = f"{name} ctas={ctas} k={k}"
                assert_same(nv, want_nv[qidx], tag + ": n_valid")
                assert_same(idx, want_idx[qidx], tag + ": ids")
                assert_same(sc, want_sc[qidx], tag + ": scores")
                if len(qidx) <= CHUNK:
                    assert_same(e.debug_fact_minmax(), mm[qidx], tag + ": mm_fact")
                assert st["stage_a_fallbacks"] == fallbacks, f"{tag}: {st['stage_a_fallbacks']} fallbacks"
                h2d.append(st["h2d_bytes"])
    finally:
        e.debug_sim_ctas(0)
    return h2d


def lo_host_extra(model):
    """h2d bytes of the lo-on-host call beyond the resident call's (both upload the queries once): the gathered lo
    rows, and per fallen-back chunk the whole lo plane streamed once more and the chunk's fp32 queries uploaded again
    (fact_stream.cu lo_host_screened_stage_a).  None where a query overflows its own caps (its gathered rows then
    depend on the order of the kernel's atomics) -- there only the lower bound is returned."""
    stream = sum(F * D * 2 + c["nb"] * D * 4 for c in model["chunks"] if c["flagged"])
    exact = all(c["exact"] for c in model["chunks"])
    gathered = sum(c["gathered"] for c in model["chunks"] if c["exact"]) * D * 2
    return stream + gathered, exact


@pytest.mark.gpu
@pytest.mark.parametrize("name", SINGLE)
def test_screen_cap_case(hb, name):
    """One case on resident planes and with the lo plane on the host: both against the oracle with the model's
    fallback count, and the lo bytes the host placement reads equal to the model's gathered rows."""
    world, _ = CASES[name]
    m = case_model(name)
    res, lo = _engine(hb, world(), False), _engine(hb, world(), True)
    try:
        h_res = _run(res, world, name, m["fallbacks"])
        h_lo = _run(lo, world, name, m["fallbacks"])
    finally:
        res.close()
        lo.close()
    want, exact = lo_host_extra(m)
    for a, b in zip(h_lo, h_res):
        if exact:
            assert a - b == want, (name, a - b, want)
        else:
            assert want < a - b < want + F * D * 2, (name, a - b, want)


@pytest.mark.gpu
@pytest.mark.parametrize("lo_host", [False, True], ids=["resident", "lo on host"])
def test_chunks_and_state(hb, lo_host):
    """2,500 queries (chunks of 1,024, 1,024 and 452) of which only chunk 1 lists 257 candidates for one query:
    exactly one fallback, every row exact.  Then a call on the same handle with every chunk at the candidate cap:
    no fallback, exact -- the flagged chunk leaves neither the other chunks nor the next call behind."""
    w = world_candidates()
    e = _engine(hb, w, lo_host)
    ref = _engine(hb, w, False) if lo_host else None
    try:
        for name in ("three chunks, one past cap", "three chunks at cap"):
            m = case_model(name)
            assert [c["nb"] for c in m["chunks"]] == [1024, 1024, 452]
            assert [c["flagged"] for c in m["chunks"]] == ([False, True, False] if "past" in name else [False] * 3)
            h = _run(e, world_candidates, name, m["fallbacks"], ks=(5, 8))
            if lo_host:
                h_ref = _run(ref, world_candidates, name, m["fallbacks"], ks=(5, 8))
                want, exact = lo_host_extra(m)
                for a, b in zip(h, h_ref):
                    assert (a - b == want) if exact else (want < a - b < want + F * D * 2), (name, a - b, want)
    finally:
        e.close()
        if ref is not None:
            ref.close()


@pytest.mark.gpu
def test_retrieve_resident_one_chunk_falls_back(hb):
    """retrieve_resident over chunks of 1,024 queries with 120 exact copies of one fact in 12 tiles (more saturated
    tiles than a query may have) and query 1,500, in chunk 1, at that fact: exactly one fallback, whose gated exact
    path runs on the overlap stream, and the passage ids and scores of the same call under the exact stage A."""
    import torch
    from hipporag_b200 import synth
    kg = synth.make_kg(30_000, 300_000, seed=21)
    assert kg.n_facts >= 65_536 + 16 * 256
    dim = 256
    fe = synth.unit_rows(kg.n_facts, dim, seed=22)
    copies = np.concatenate([np.arange(t * 256, t * 256 + 10) for t in range(4, 16)])
    fe[copies] = fe[1024]
    pe = synth.unit_rows(kg.n_pass, dim, seed=23)
    qf, qp, j = synth.make_queries(kg, fe, pe, 2100, seed=24)
    near = np.isin(j, np.r_[copies, 1024])                 # queries built on a copy would tie as well
    qf[near], qp[near] = qf[~near][0], qp[~near][0]
    qf[1500] = fe[1024]
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
        (i0, s0, fb), (i1, s1, fb_exact) = outs
        assert fb == 1 and fb_exact == 0, (fb, fb_exact)
        assert np.array_equal(i0, i1)
        assert np.array_equal(s0.view(np.uint32), s1.view(np.uint32))
    finally:
        e.close()
