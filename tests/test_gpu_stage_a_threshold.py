"""The fused stage-A epilogue under its per-query bound, on exact scores.

k_sim_tc's fused epilogue keeps, per (query, 256-fact tile), only the keys that reach a per-query bound: the largest
8th-best key of any tile list written so far.  The bound depends on the order in which the persistent CTAs visit the
tiles, so these cases are run at several CTA counts; the selected facts, their min-max scores and n_valid must equal the
float32 oracle bit for bit whatever the order.  Scores are exact (small integers / 4, see test_gpu_selection_exact).
"""
import numpy as np
import pytest

from tests.test_gpu_selection_exact import (as_f32, assert_same, exact_ints, expected_topk, minmax32, ranking,
                                            raw_scores)

M, DIM, TILE = 2900, 40, 256          # 12 fact tiles, the last one ragged (84 columns)


def _row_with_sum(s, dim):
    """An integer row in [-3, 3]^dim whose entries sum to s (|s| <= 3 dim)."""
    r = np.zeros(dim, np.int64)
    a, sign = abs(int(s)), 1 if s >= 0 else -1
    r[:a // 3] = 3 * sign
    if a % 3:
        r[a // 3] = (a % 3) * sign
    return r


def _case(kind, rng):
    """(Ei, q): the fact rows and the planted query of one case."""
    if kind == "rising":
        # the planted query's scores rise along the fact axis in runs of ties: the bound climbs tile after tile
        q = np.full(DIM, 3, np.int64)
        levels = np.round(np.linspace(-3 * DIM, 3 * DIM, M)).astype(np.int64)
        return np.stack([_row_with_sum(s, DIM) for s in levels]), q
    if kind in ("tie_8_9", "late_tile"):
        q = np.zeros(DIM, np.int64)
        q[:8] = 3
        Ei = exact_ints(rng, (M, DIM))
        Ei[:, :8] = np.minimum(Ei[:, :8], 2)             # every other row scores <= 3 * 16 / 16
        if kind == "tie_8_9":
            # the 7 best in tile 0; the 8th and 9th best tie exactly, in tiles 2 and 4 (the lower index wins)
            Ei[3:10, :8] = 3
            for r in (2 * TILE + 5, 5 * TILE - 100):
                Ei[r, :8] = 3
                Ei[r, 0] = 2
        else:
            # three runners-up in tile 0 raise the bound early; the whole top 8 sits in tile 10 (the last full one)
            Ei[[1, 2, 3], :8] = 3
            Ei[[1, 2, 3], 0] = 2
            top = 10 * TILE + rng.choice(TILE, 8, replace=False)
            Ei[top, :8] = 3
        return Ei, q
    if kind == "all_negative":
        return exact_ints(rng, (M, DIM), 1, 3), -exact_ints(rng, DIM, 1, 3)
    if kind == "all_equal":
        return np.repeat(exact_ints(rng, (1, DIM)), M, axis=0), exact_ints(rng, DIM)
    raise ValueError(kind)


KINDS = ("rising", "tie_8_9", "late_tile", "all_negative", "all_equal")


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


@pytest.mark.gpu
@pytest.mark.parametrize("n_ctas", [1, 7, 0], ids=["ctas1", "ctas7", "num_sms"])
@pytest.mark.parametrize("B", [129, 1100])
@pytest.mark.parametrize("kind", KINDS)
def test_fused_stage_a_bound_is_exact(hb, kind, B, n_ctas):
    rng = np.random.default_rng(KINDS.index(kind) * 1009 + B)
    Ei, q = _case(kind, rng)
    Qi = exact_ints(rng, (B, DIM))
    if kind == "all_negative":
        Qi = -exact_ints(rng, (B, DIM), 1, 3)
    planted = [r for r in (0, 127, 128, 1023, 1024, B - 1) if r < B]   # both query tiles, both 1024-query chunks
    Qi[planted] = q
    if kind == "all_equal":
        Qi[1] = 0                                        # the zero query: every score 0.0
    raw = raw_scores(Qi, Ei)
    order = ranking(raw)
    # the planted structure is there
    if kind == "rising":
        assert np.all(np.diff(raw[0]) >= 0) and raw[0].max() > raw[0, :TILE].max()
    elif kind == "tie_8_9":
        assert raw[0, order[0, 7]] == raw[0, order[0, 8]] > raw[0, order[0, 9]]
        assert order[0, 7] // TILE == 2 and order[0, 8] // TILE == 4 and order[0, 6] // TILE == 0
    elif kind == "late_tile":
        assert np.all(order[0, :8] // TILE == 10) and raw[0, order[0, 7]] > raw[0, order[0, 8]]
    elif kind == "all_negative":
        assert raw.max() < 0
    else:
        assert np.all(raw == raw[:, :1])
    norm = minmax32(raw)
    e = hb.Engine(0)
    e.load_embeddings(as_f32(Ei), as_f32(np.ones((4, DIM), np.int64)))
    e.debug_sim_ctas(n_ctas)
    try:
        for mode in (hb.SIM_BF16X3, hb.SIM_BF16):
            e.set_options(sim_mode=mode)
            for k in range(1, 9):
                idx, sc, nv = e.stage_a(as_f32(Qi), k)
                want_idx, want_sc, want_nv = expected_topk(norm, order, k)
                tag = f"{kind} B={B} n_ctas={n_ctas} mode={mode} k={k}"
                assert_same(nv, want_nv, tag + ": n_valid")
                assert_same(idx, want_idx, tag + ": ids")
                assert_same(sc, want_sc, tag + ": scores")
    finally:
        e.close()
