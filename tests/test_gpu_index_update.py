"""In-place index updates (hrag_index_append / hrag_index_delete) against fresh loads, bit for bit.

Every case applies the update to a mutable handle and, in numpy, to the arrays it was loaded from; a fresh mutable
handle then loads the resulting arrays (load_graph COO, load_tables, load_embeddings).  The two must agree byte for
byte: every graph plane (hrag_debug_graph), every table, embedding and edge-list plane (hrag_debug_index), and the
outputs of every entry that reads them -- stage A (k = 5, 16), stage B (fp32 solver at B = 8, mixed at B = 40),
float64 stage B, ppr, ppr_f64, topk_similarity, knn_threshold and retrieve_resident over two chunks.
"""
from dataclasses import dataclass, replace

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DIM = 64
GRAPH_PLANES = ("row_ptr", "cv", "val_lo", "row_order", "long_rows", "long_seg_ptr", "segs")
INDEX_PLANES = ("passage_vid", "fact_subj_vid", "fact_obj_vid", "ent_chunk_count", "fact_hi", "fact_lo",
                "passage_hi", "passage_lo", "fact_f32", "passage_f32", "edge_src", "edge_dst", "edge_w")


@dataclass
class Index:
    """The arrays a fresh load takes."""
    n: int
    src: np.ndarray
    dst: np.ndarray
    w: np.ndarray
    pv: np.ndarray
    fs: np.ndarray
    fo: np.ndarray
    cc: np.ndarray
    fe: np.ndarray
    pe: np.ndarray


def _base(seed=3, n_nodes=6000, n_edges=60000):
    """A power-law graph (hub rows far over 256 non-zeros) with one entity whose only neighbour is passage 3."""
    from hipporag_b200 import synth
    kg = synth.make_kg(n_nodes, n_edges, seed=seed, topology="powerlaw")
    lonely = kg.n_ent - 1                                   # make_kg leaves the last entities isolated
    src = np.r_[kg.edge_src, lonely].astype(np.int32)
    dst = np.r_[kg.edge_dst, kg.passage_vid[3]].astype(np.int32)
    w = np.r_[kg.edge_w, 1.0]
    return Index(kg.n_nodes, src, dst, w, kg.passage_vid.copy(), kg.fact_subj_vid.copy(), kg.fact_obj_vid.copy(),
                 kg.ent_chunk_count.copy(), synth.unit_rows(kg.n_facts, DIM, seed + 1),
                 synth.unit_rows(kg.n_pass, DIM, seed + 2))


@dataclass
class Batch:
    n_new: int
    src: np.ndarray
    dst: np.ndarray
    w: np.ndarray
    pv: np.ndarray
    fs: np.ndarray
    fo: np.ndarray
    cc: np.ndarray          # the whole new table
    fe: np.ndarray
    pe: np.ndarray


def _batch(ix: Index, rng, n_ent=30, n_pass=6, n_edges=400, n_facts=40):
    """An append: new entities (some isolated) and passages, edges among old and new vertices, parallel copies of old
    edges, edges between old vertices only, w <= 0 / NaN edges, new facts (some with an absent end) and a changed
    chunk count of an old entity."""
    n0, n_new = ix.n, n_ent + n_pass
    N = n0 + n_new
    live_new = n0 + np.arange(n_ent - min(5, n_ent // 3))   # the last new entities stay isolated
    pv = (n0 + n_ent + np.arange(n_pass)).astype(np.int32)
    a = rng.choice(np.r_[live_new, pv], n_edges)
    b = rng.integers(0, n0, n_edges)
    par = rng.integers(0, ix.src.size, 50)                  # parallel copies of existing edges
    old_a, old_b = rng.integers(0, n0, 60), rng.integers(0, n0, 60)
    src = np.r_[a, ix.src[par], old_a, [pv[0], pv[-1], live_new[0]]].astype(np.int32)
    dst = np.r_[b, ix.dst[par], old_b, [live_new[-1], 5, 7]].astype(np.int32)
    w = np.r_[rng.uniform(0.1, 2.0, n_edges), rng.uniform(0.1, 2.0, 50), rng.uniform(0.1, 2.0, 60),
              [0.0, -1.0, np.nan]]
    ents = np.r_[live_new, rng.integers(0, n0 - len(ix.pv), 20)]
    fs = rng.choice(ents, n_facts).astype(np.int32)
    fo = rng.choice(ents, n_facts).astype(np.int32)
    fo[:3] = -1
    cc = np.r_[ix.cc, rng.integers(0, 4, n_new)].astype(np.int32)
    cc[pv] = 0
    cc[int(np.argmax(ix.cc))] += 7                          # an old entity's chunk count changes
    return Batch(n_new, src, dst, w, pv, fs, fo, cc, rng.standard_normal((n_facts, DIM)).astype(np.float32),
                 rng.standard_normal((n_pass, DIM)).astype(np.float32))


def _appended(ix: Index, bt: Batch) -> Index:
    return Index(ix.n + bt.n_new, np.r_[ix.src, bt.src], np.r_[ix.dst, bt.dst], np.r_[ix.w, bt.w],
                 np.r_[ix.pv, bt.pv], np.r_[ix.fs, bt.fs], np.r_[ix.fo, bt.fo], bt.cc,
                 np.concatenate([ix.fe, bt.fe]), np.concatenate([ix.pe, bt.pe]))


def _deleted(ix: Index, nodes, facts) -> Index:
    keep = np.ones(ix.n, bool)
    keep[nodes] = False
    vmap = np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int32)
    ke = keep[ix.src] & keep[ix.dst]
    kp = keep[ix.pv]
    kf = np.ones(ix.fs.size, bool)
    kf[facts] = False

    def rel(v):
        return np.where(v >= 0, vmap[np.maximum(v, 0)], -1).astype(np.int32)
    return Index(int(keep.sum()), vmap[ix.src[ke]], vmap[ix.dst[ke]], ix.w[ke], vmap[ix.pv[kp]], rel(ix.fs[kf]),
                 rel(ix.fo[kf]), ix.cc[keep], ix.fe[kf], ix.pe[kp])


def _engine(ix: Index, mutable=True):
    from hipporag_b200 import Engine
    e = Engine(0, mutable=mutable)
    e.load_graph(ix.n, ix.src, ix.dst, ix.w)
    e.load_tables(ix.pv, ix.fs, ix.fo, ix.cc)
    e.load_embeddings(ix.fe, ix.pe)
    return e


def _append(e, bt: Batch):
    e.append(bt.n_new, bt.src, bt.dst, bt.w, bt.pv, bt.fs, bt.fo, bt.cc, bt.fe, bt.pe)


def _delete(e, ix: Index, nodes, facts):
    keep = np.ones(ix.n, bool)
    keep[nodes] = False
    e.delete(np.asarray(nodes, np.int32), np.asarray(facts, np.int32), ix.cc[keep])


def _planes(e):
    return ({p: e.debug_graph(p) for p in GRAPH_PLANES}, {p: e.debug_index(p) for p in INDEX_PLANES})


def _assert_planes_equal(a, b):
    (ga, ia), (gb, ib) = _planes(a), _planes(b)
    for p in GRAPH_PLANES:
        assert ga[p].tobytes() == gb[p].tobytes(), f"graph plane {p}"
    for p in INDEX_PLANES:
        assert ia[p].tobytes() == ib[p].tobytes(), f"index plane {p}"
    assert (a.n_nodes, a.n_passages, a.n_facts) == (b.n_nodes, b.n_passages, b.n_facts)


def _outputs(e, seed=9):
    import torch
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((1025, DIM)).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)           # cosines ~ N(0, 1/8): few rows clear the knn threshold
    qp = rng.standard_normal((1025, DIM)).astype(np.float32)
    out = {}
    out["a5"] = e.stage_a(q[:40], 5)
    out["a16"] = e.stage_a(q[:40], 16)
    idx, score, _ = out["a5"]
    out["b8"] = e.stage_b(qp[:8], idx[:8], score[:8], topk=50)
    out["b40"] = e.stage_b(qp[:40], idx, score, topk=50)
    out["b_f64"] = e.stage_b_f64(qp[:8], idx[:8], score[:8], topk=50)
    reset = np.abs(rng.standard_normal((4, e.n_nodes)))
    out["ppr"] = e.ppr(reset.astype(np.float32))
    out["ppr_f64"] = e.ppr_f64(reset)
    out["topk_f"] = e.topk_similarity(0, q[:16], 30)
    out["topk_p"] = e.topk_similarity(1, qp[:16], 30)
    out["knn"] = e.knn_threshold(0, q[:16], 0.3, 512)
    assert out["knn"][2].max() <= 512                       # no candidate list overflowed
    dq, dp = torch.from_numpy(q).cuda(), torch.from_numpy(qp).cuda()
    ids = torch.empty((1025, 20), dtype=torch.int32, device="cuda")
    sc = torch.empty((1025, 20), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    e.retrieve_resident(dq, dp, ids, sc, topk=20)
    torch.cuda.synchronize()
    out["resident"] = (ids.cpu().numpy(), sc.cpu().numpy())
    return out


def _assert_outputs_equal(a, b):
    oa, ob = _outputs(a), _outputs(b)
    for k in oa:
        for x, y in zip(oa[k], ob[k]):
            assert np.asarray(x).tobytes() == np.asarray(y).tobytes(), f"output {k}"


def _assert_same(updated, ix: Index, outputs=True):
    fresh = _engine(ix)
    try:
        _assert_planes_equal(updated, fresh)
        if outputs:
            _assert_outputs_equal(updated, fresh)
    finally:
        fresh.close()


# ----------------------------------------------------------------------------- append
def test_append_batches_equal_a_fresh_load():
    ix = _base()
    e = _engine(ix)
    assert np.diff(e.debug_graph("row_ptr")).max() > 256
    rng = np.random.default_rng(1)
    for i in range(3):
        bt = _batch(ix, rng)
        _append(e, bt)
        ix = _appended(ix, bt)
        _assert_same(e, ix, outputs=i == 2)
    e.close()


def test_append_from_device_tensors():
    import torch
    ix = _base(seed=4, n_nodes=3000, n_edges=20000)
    e = _engine(ix)
    bt = _batch(ix, np.random.default_rng(2))
    cuda = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (bt.src, bt.dst, bt.w, bt.fe, bt.pe)]
    e.append(bt.n_new, cuda[0], cuda[1], cuda[2], bt.pv, bt.fs, bt.fo, bt.cc, cuda[3], cuda[4])
    _assert_same(e, _appended(ix, bt), outputs=False)
    e.close()


# ----------------------------------------------------------------------------- delete
def test_delete_equals_a_fresh_load():
    ix = _base()
    e = _engine(ix)
    deg = np.bincount(np.r_[ix.src, ix.dst], minlength=ix.n)
    hub = int(np.argmax(deg))
    assert deg[hub] > 512                                   # its row is cut into segments
    lonely = int(ix.src[-1])                                # its only neighbour is passage 3
    nodes = sorted({0, hub, ix.n - 1, int(ix.pv[3])})
    dead = np.zeros(ix.n, bool)
    dead[nodes] = True
    survivors = np.flatnonzero(~dead[ix.fs] & ~dead[np.maximum(ix.fo, 0)])
    facts = np.sort(survivors[::7][:40])
    _delete(e, ix, nodes, facts)
    ix = _deleted(ix, nodes, facts)
    lonely_new = lonely - int(np.sum(np.asarray(nodes) < lonely))
    assert np.diff(e.debug_graph("row_ptr"))[lonely_new] == 0   # the entity is isolated now
    _assert_same(e, ix)
    e.close()


def test_delete_that_shrinks_n_does_not_replay_a_stale_solve():
    """A mixed stage B captures its solve graphs; a delete of one vertex then shrinks N and the next mixed stage B
    must solve the new graph."""
    ix = _base(seed=5, n_nodes=4000, n_edges=40000)
    e = _engine(ix)
    rng = np.random.default_rng(3)
    qf = rng.standard_normal((40, DIM)).astype(np.float32)
    qp = rng.standard_normal((40, DIM)).astype(np.float32)
    idx, score, _ = e.stage_a(qf, 5)
    e.stage_b(qp, idx, score, topk=30)
    nodes = [int(ix.n - 2)]
    _delete(e, ix, nodes, [])
    ix = _deleted(ix, nodes, [])
    fresh = _engine(ix)
    idx, score, _ = fresh.stage_a(qf, 5)
    for a, b in zip(e.stage_b(qp, idx, score, topk=30), fresh.stage_b(qp, idx, score, topk=30)):
        assert a.tobytes() == b.tobytes()
    fresh.close()
    e.close()


# ----------------------------------------------------------------------------- interleaved, capacity growth
def test_interleaved_updates_and_reserve():
    ix0 = _base(seed=6, n_nodes=300, n_edges=2000)         # small, so the appends below outgrow it several times
    rng = np.random.default_rng(4)
    ops, ix = [], ix0
    bt = _batch(ix, rng, n_edges=200)
    ops.append(("append", bt))
    ix = _appended(ix, bt)
    nodes, facts = sorted({1, 17, int(ix.pv[2]), ix.n - 3}), [0, 5, 9]
    ops.append(("delete", (ix, nodes, facts)))
    ix = _deleted(ix, nodes, facts)
    for _ in range(12):     # 12 appends: the edge list, passage and fact planes each grow by half several times
        bt = _batch(ix, rng, n_ent=4, n_pass=6, n_edges=200, n_facts=20)
        ops.append(("append", bt))
        ix = _appended(ix, bt)

    def run(e):
        for kind, arg in ops:
            _append(e, arg) if kind == "append" else _delete(e, *arg)

    grown, reserved = _engine(ix0), _engine(ix0)
    reserved.reserve(nodes=ix.n + 100, edges=ix.src.size + 1000, facts=ix.fs.size + 50, passages=ix.pv.size + 10)
    run(grown)
    run(reserved)
    _assert_same(grown, ix)
    _assert_planes_equal(grown, reserved)
    _assert_outputs_equal(grown, reserved)
    grown.close()
    reserved.close()


# ----------------------------------------------------------------------------- call contract
def _snapshot(e):
    g, i = _planes(e)
    return {**{"g_" + k: v.tobytes() for k, v in g.items()}, **{"i_" + k: v.tobytes() for k, v in i.items()},
            "sizes": (e.n_nodes, e.n_passages, e.n_facts)}


def test_rejected_calls_leave_the_handle_unchanged():
    import torch
    from hipporag_b200 import HragError
    ix = _base(seed=7, n_nodes=2000, n_edges=15000)
    e = _engine(ix)
    before = _snapshot(e)
    bt = _batch(ix, np.random.default_rng(5))
    N = ix.n + bt.n_new
    bad = replace(bt, dst=np.r_[bt.dst[:-1], N].astype(np.int32))
    with pytest.raises(HragError, match="out of range"):
        _append(e, bad)
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (bad.src, bad.dst, bad.w)]
    with pytest.raises(HragError, match="out of range"):
        e.append(bad.n_new, *dev, bt.pv, bt.fs, bt.fo, bt.cc, bt.fe, bt.pe)
    with pytest.raises(HragError, match="out of range"):
        _append(e, replace(bt, pv=np.r_[bt.pv[:-1], N].astype(np.int32)))
    keep_cc = ix.cc[:-2]
    with pytest.raises(HragError, match="sorted, unique"):
        e.delete(np.array([9, 4], np.int32), np.zeros(0, np.int32), keep_cc)
    with pytest.raises(HragError, match="sorted, unique"):
        e.delete(np.array([4, 4], np.int32), np.zeros(0, np.int32), keep_cc)
    with pytest.raises(HragError, match="sorted, unique"):
        e.delete(np.zeros(0, np.int32), np.array([3, 3], np.int32), ix.cc)
    with pytest.raises(HragError, match="dim"):
        _append(e, replace(bt, fe=np.zeros((bt.fs.size, DIM + 8), np.float32),
                           pe=np.zeros((bt.pv.size, DIM + 8), np.float32)))
    assert _snapshot(e) == before
    # an accepted append uploads its own inputs and nothing else
    e.reset_stats()
    _append(e, bt)
    new_bytes = sum(a.nbytes for a in (bt.src, bt.dst, bt.w, bt.pv, bt.fs, bt.fo, bt.cc, bt.fe, bt.pe))
    assert e.stats()["h2d_bytes"] == new_bytes
    e.close()


def test_handles_that_cannot_be_updated():
    import torch
    from hipporag_b200 import Engine, HragError
    from hipporag_b200.engine import build_transition_csr
    ix = _base(seed=8, n_nodes=2000, n_edges=15000)
    bt = _batch(ix, np.random.default_rng(6))
    e = _engine(ix, mutable=False)
    before = _snapshot(e)
    with pytest.raises(HragError, match="not mutable"):
        _append(e, bt)
    assert _snapshot(e) == before
    e.close()
    e = Engine(0, mutable=True)
    e.load_graph_csr(ix.n, *build_transition_csr(ix.n, ix.src, ix.dst, ix.w, dtype=np.float64))
    e.load_tables(ix.pv, ix.fs, ix.fo, ix.cc)
    e.load_embeddings(ix.fe, ix.pe)
    before = _snapshot(e)
    with pytest.raises(HragError, match="keeps no edge list"):
        _append(e, bt)
    with pytest.raises(HragError, match="keeps no edge list"):
        _delete(e, ix, [3], [])
    assert _snapshot(e) == before
    e.close()
    e = Engine(0, mutable=True)
    e.load_graph(ix.n, ix.src, ix.dst, ix.w)
    e.load_tables(ix.pv, ix.fs, ix.fo, ix.cc)
    fe, pe = torch.from_numpy(ix.fe).cuda(), torch.from_numpy(ix.pe).cuda()
    e.load_embeddings(fe, pe)
    before = _snapshot(e)
    with pytest.raises(HragError, match="borrowed"):
        _append(e, bt)
    with pytest.raises(HragError, match="borrowed"):
        _delete(e, ix, [3], [])
    assert _snapshot(e) == before
    e.close()


# ----------------------------------------------------------------------------- other embedding layouts
def _engine_layout(ix: Index, layout: str):
    """'streamed': bf16 planes only (load_embeddings_streamed); 'fp32_only': dim % 8 != 0, so no bf16 planes."""
    from hipporag_b200 import Engine
    e = Engine(0, mutable=True)
    e.load_graph(ix.n, ix.src, ix.dst, ix.w)
    e.load_tables(ix.pv, ix.fs, ix.fo, ix.cc)
    if layout == "streamed":
        for which, m in ((0, ix.fe), (1, ix.pe)):
            e.load_embeddings_streamed(which, m.shape[0], m.shape[1], [(0, m[:100]), (100, m[100:])])
        e.n_passages = ix.pv.size
    else:
        e.load_embeddings(ix.fe, ix.pe)
    return e


@pytest.mark.parametrize("layout", ["streamed", "fp32_only"])
def test_updates_with_other_embedding_layouts(layout):
    """Appends and deletes keep only the planes a fresh load of that layout holds: the bf16 planes of a streamed
    matrix (no fp32 rows), the fp32 rows of a dim % 8 != 0 matrix (no bf16 planes)."""
    ix = _base(seed=9, n_nodes=2000, n_edges=15000)
    cut = (lambda m: np.ascontiguousarray(m[:, :60])) if layout == "fp32_only" else (lambda m: m)
    ix = replace(ix, fe=cut(ix.fe), pe=cut(ix.pe))
    e = _engine_layout(ix, layout)
    rng = np.random.default_rng(7)
    bt = _batch(ix, rng)
    bt = replace(bt, fe=cut(bt.fe), pe=cut(bt.pe))
    _append(e, bt)
    ix = _appended(ix, bt)
    nodes, facts = sorted({2, int(ix.pv[1]), ix.n - 1}), [1, 8]
    _delete(e, ix, nodes, facts)
    ix = _deleted(ix, nodes, facts)
    fresh = _engine_layout(ix, layout)
    _assert_planes_equal(e, fresh)
    planes = fresh.debug_index("fact_f32", size_only=True), fresh.debug_index("fact_hi", size_only=True)
    assert (planes[0] == 0) if layout == "streamed" else (planes[1] == 0)
    rng = np.random.default_rng(8)
    q = rng.standard_normal((40, ix.fe.shape[1])).astype(np.float32)
    for eng_out in zip(*[(x.stage_a(q, 5), x.topk_similarity(1, q, 20)) for x in (e, fresh)]):
        for a, b in zip(*eng_out):
            assert a.tobytes() == b.tobytes()
    idx, score, _ = fresh.stage_a(q, 5)
    for B in (8, 40):
        for a, b in zip(e.stage_b(q[:B], idx[:B], score[:B], topk=30), fresh.stage_b(q[:B], idx[:B], score[:B], topk=30)):
            assert a.tobytes() == b.tobytes()
    e.close()
    fresh.close()
