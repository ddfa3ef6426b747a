"""Reloading the graph or the tables of a live handle (Engine reuse across index() / delete()).

A rejected load must leave the handle exactly as it was: the same graph, tables, solver state and captured solves, so
every earlier result comes back bit for bit.  A successful reload of a different graph with the same vertex count must
invalidate the captured mixed-precision solves: the next solve equals a fresh handle's on that graph bit for bit.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIM = 64
HUB_DEG = 600          # one row above the 256-non-zero long-row cut, so the reload replaces the segment tables too


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def _kg(seed, hub_deg=HUB_DEG):
    from hipporag_b200 import synth
    kg = synth.make_kg(4000, 40000, seed=seed)
    rng = np.random.default_rng(seed)
    hub = rng.choice(np.arange(1, kg.n_nodes), hub_deg, replace=False).astype(np.int32)
    src = np.concatenate([kg.edge_src, np.zeros(hub_deg, np.int32)])
    dst = np.concatenate([kg.edge_dst, hub])
    w = np.concatenate([kg.edge_w, rng.uniform(0.5, 2.0, hub_deg)])
    return kg, src, dst, w


def _engine(hb, kg, src, dst, w):
    from hipporag_b200 import synth
    e = hb.Engine(0)
    e.load_graph(kg.n_nodes, src, dst, w)      # COO ingest: keeps the fp64 plane ppr_f64 needs
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    e.load_embeddings(synth.unit_rows(kg.n_facts, DIM, seed=1), synth.unit_rows(kg.n_pass, DIM, seed=2))
    return e


def _resets(n, b, seed):
    rng = np.random.default_rng(seed)
    r = np.zeros((b, n), np.float32)
    for i in range(b):
        r[i, rng.choice(n, 5, replace=False)] = rng.uniform(0.1, 1.0, 5)
    return r


def _results(e, kg):
    """fp32 solve (B = 4), mixed solve (B = 40), fp64 solve and a mixed-precision stage B (B = 40)."""
    from hipporag_b200 import synth
    fe = synth.unit_rows(kg.n_facts, DIM, seed=1)
    pe = synth.unit_rows(kg.n_pass, DIM, seed=2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 40, seed=3)
    idx, score, _ = e.stage_a(qf, k=5)
    ids, scores = e.stage_b(qp, idx, score)
    return dict(fp32=e.ppr(_resets(kg.n_nodes, 4, 4)), mixed=e.ppr(_resets(kg.n_nodes, 40, 5)),
                f64=e.ppr_f64(_resets(kg.n_nodes, 4, 6).astype(np.float64)), stage_b_ids=ids, stage_b_scores=scores)


def _assert_same(got, want, what):
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, (what, k)
        assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), f"{what}: {k} changed"


def test_rejected_reload_keeps_the_handle(hb):
    kg, src, dst, w = _kg(7)
    e = _engine(hb, kg, src, dst, w)
    want = _results(e, kg)
    _assert_same(_results(e, kg), want, "repeat")    # replayed solves reproduce the captured ones
    n = kg.n_nodes
    row_ptr, col, val = hb.build_transition_csr(n, src, dst, w, dtype=np.float64)

    bad_col = col.copy()
    bad_col[len(bad_col) // 2] = n
    non_monotone = row_ptr.copy()
    k = int(np.argmax(np.diff(row_ptr) >= 2)) + 1   # a row_ptr entry inside the range, moved past its successor
    non_monotone[k] = row_ptr[k + 1] + 1
    bad_edges = dst.copy()
    bad_edges[3] = n
    bad_pv = np.array(kg.passage_vid, np.int32)
    bad_pv[-1] = n
    rejected = [
        ("column out of range (fp64 CSR)", lambda: e.load_graph_csr(n, row_ptr, bad_col, val)),
        ("column out of range (fp32 CSR)", lambda: e.load_graph_csr(n, row_ptr, bad_col, val.astype(np.float32))),
        ("row_ptr not monotone", lambda: e.load_graph_csr(n, non_monotone, col, val)),
        ("edge endpoint out of range (COO)", lambda: e.load_graph(n, src, bad_edges, w)),
        ("passage_vid out of range", lambda: e.load_tables(bad_pv, kg.fact_subj_vid, kg.fact_obj_vid,
                                                           kg.ent_chunk_count)),
    ]
    for what, load in rejected:
        with pytest.raises(hb.HragError):
            load()
        _assert_same(_results(e, kg), want, f"after a rejected load ({what})")
    e.close()


def test_reload_invalidates_captured_solves(hb):
    kg, src, dst, w = _kg(7)
    e = _engine(hb, kg, src, dst, w)
    resets = _resets(kg.n_nodes, 40, 8)
    first = e.ppr(resets)                            # captures the mixed solve for this buffer set and plan
    # another graph on the same N with other edges, non-zero count and long-row segments (a hub of 900 non-zeros is
    # 4 segments, one of 600 is 3), so a stale captured solve could not give this graph's result by accident
    kg2, src2, dst2, w2 = _kg(8, hub_deg=900)
    assert kg2.n_nodes == kg.n_nodes
    e.load_graph(kg2.n_nodes, src2, dst2, w2)
    got = e.ppr(resets)
    fresh = _engine(hb, kg2, src2, dst2, w2)
    want = fresh.ppr(resets)
    assert not np.array_equal(first, want)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    fresh.close()
    e.close()
