"""The resident self-KNN index (hrag_knn_index_update / _read): after every update of a sequence it must hold, bit for
bit, what a fresh handle's threshold KNN (hrag_knn_threshold, with the rows whose candidates overflow 512 redone through
hrag_topk_similarity, as knn.retrieve_knn does) gives over the current rows.

Rows are +-1 in d = 64, so the unit rows are +-1/8 and every score is an exact multiple of 1/64: ties are everywhere,
across tiles and across the boundary between kept and new rows.  Planted clusters share 48 coordinates with a template
(score >= 0.5 among themselves), so some rows have more than 128 and some more than 512 neighbours >= the threshold.
"""
import numpy as np
import pytest

DIM = 64
THR = 24 / 64            # exact in float32: the GEMM's cut and the redo's cut agree
KMAX = 128


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


def _rows(rng, n, template=None):
    x = rng.choice([-1.0, 1.0], size=(n, DIM)).astype(np.float32)
    if template is not None:
        x[:, :48] = template[:48]
    return x / np.float32(8)


def per_call(hb, keys, thr=THR, kmax=KMAX):
    """(ids, scores) [rows, kmax] of a fresh handle's threshold KNN + overflow redo over `keys` (knn.py's recipe)."""
    M = keys.shape[0]
    if M == 0:
        return np.zeros((0, kmax), np.int32), np.zeros((0, kmax), np.float32)
    e = hb.Engine(0)
    try:
        e.load_embeddings(keys, keys[:1])
        ids, sc, found = e.knn_threshold(0, keys, thr, kmax)
        redo = np.nonzero(found > 512)[0]
        if redo.size:
            rid, rsc = e.topk_similarity(0, keys[redo], int(min(kmax, M)))
            for j, q in enumerate(redo):
                keep = rsc[j] >= np.float32(thr)
                ids[q], sc[q] = -1, 0.0
                ids[q, :keep.sum()] = rid[j][keep]
                sc[q, :keep.sum()] = rsc[j][keep]
        return ids, sc
    finally:
        e.close()


def assert_index(hb, eng, keys, thr=THR, kmax=KMAX, what=""):
    ids, sc = eng.knn_index_read()
    want_ids, want_sc = per_call(hb, keys, thr, kmax)
    assert ids.shape == want_ids.shape, what
    bad = np.nonzero((ids != want_ids).any(axis=1) | (sc.view(np.uint32) != want_sc.view(np.uint32)).any(axis=1))[0]
    assert bad.size == 0, f"{what}: {bad.size} rows differ, first {bad[:5]}"
    return want_ids


class Store:
    """Keys and rows changed the way EmbeddingStore changes them: appends, in-order deletes."""

    def __init__(self, rows):
        self.rows = rows
        self.keys = list(range(rows.shape[0]))
        self.next = rows.shape[0]

    def change(self, delete=(), append=None):
        keep = np.ones(len(self.keys), bool)
        keep[list(delete)] = False
        kept_from = np.flatnonzero(keep)
        self.rows = self.rows[keep]
        self.keys = [k for k, s in zip(self.keys, keep) if s]
        if append is not None and append.shape[0]:
            self.rows = np.concatenate([self.rows, append])
            self.keys += list(range(self.next, self.next + append.shape[0]))
            self.next += append.shape[0]
        return kept_from


@pytest.mark.gpu
def test_update_sequence_equals_fresh_all_pairs(hb):
    rng = np.random.default_rng(11)
    ta, tb = rng.choice([-1.0, 1.0], DIM), rng.choice([-1.0, 1.0], DIM)
    base = np.concatenate([_rows(rng, 1500), _rows(rng, 560, ta), _rows(rng, 200, tb), _rows(rng, 500)])
    base[1700] = base[3]                                   # exact duplicate: a tie broken by row
    st = Store(base[rng.permutation(base.shape[0])])
    eng = hb.Engine(0)
    assert eng.knn_index_update(st.rows, None, THR, KMAX) == 0
    lists = assert_index(hb, eng, st.rows, what="build")
    counts = (st.rows @ st.rows.T >= np.float32(THR)).sum(axis=1)
    assert (counts > 512).any() and ((counts > 128) & (counts <= 512)).any() and (counts == 1).any()

    # append only: duplicates of old rows (exact ties across the boundary) and 600 new members of cluster A, so the
    # old members' candidates among the new keys alone overflow 512 (old x new redo), as do the new members' (new x all)
    dup = st.rows[rng.choice(st.rows.shape[0], 20, replace=False)]
    kf = st.change(append=np.concatenate([dup, _rows(rng, 600, ta), _rows(rng, 40)]))
    assert eng.knn_index_update(st.rows, kf, THR, KMAX) == 1
    lists = assert_index(hb, eng, st.rows, what="append")

    # delete only: rows of cluster B whose lists are full (> 128 neighbours) lose a listed neighbour -> refill
    b_rows = np.flatnonzero((st.rows[:, :48] * 8 == tb[:48]).all(axis=1))
    listed = set(lists[b_rows[0]][lists[b_rows[0]] >= 0].tolist())
    victims = [r for r in b_rows[1:] if r in listed][:5] + rng.choice(st.rows.shape[0], 60, replace=False).tolist()
    kf = st.change(delete=sorted(set(victims)))
    assert eng.knn_index_update(st.rows, kf, THR, KMAX) == 1
    lists = assert_index(hb, eng, st.rows, what="delete")

    # delete of unlisted neighbours only (a B row whose list is full keeps it: no refill), then delete + append
    b_rows = np.flatnonzero((st.rows[:, :48] * 8 == tb[:48]).all(axis=1))
    listed = set(lists[b_rows[0]][lists[b_rows[0]] >= 0].tolist())
    unlisted = [r for r in b_rows if r not in listed][:3]
    assert unlisted
    kf = st.change(delete=unlisted)
    assert eng.knn_index_update(st.rows, kf, THR, KMAX) == 1
    assert_index(hb, eng, st.rows, what="delete unlisted")
    kf = st.change(delete=rng.choice(st.rows.shape[0], 100, replace=False).tolist(),
                   append=np.concatenate([_rows(rng, 30, tb), _rows(rng, 70)]))
    assert eng.knn_index_update(st.rows, kf, THR, KMAX) == 1
    assert_index(hb, eng, st.rows, what="delete + append")

    # no change: nothing is scored
    eng.reset_stats()
    assert eng.knn_index_update(st.rows, np.arange(st.rows.shape[0]), THR, KMAX) == 2
    s = eng.stats()
    assert s["ms_sim_fact"] == 0.0 and s["ms_topk"] == 0.0
    assert_index(hb, eng, st.rows, what="unchanged")

    # the same sequence from device rows
    import torch
    kf = st.change(delete=[0, 5], append=_rows(rng, 10, ta))
    assert eng.knn_index_update(torch.from_numpy(st.rows).cuda(), kf, THR, KMAX) == 1
    assert_index(hb, eng, st.rows, what="device rows")

    # deleting every key
    kf = st.change(delete=range(st.rows.shape[0]))
    assert eng.knn_index_update(np.zeros((0, DIM), np.float32), kf, THR, KMAX) == 1
    assert eng.knn_index_info() == (0, DIM, KMAX)
    ids, sc = eng.knn_index_read()
    assert ids.shape == (0, KMAX)
    kf = st.change(append=_rows(rng, 300, ta))
    assert eng.knn_index_update(st.rows, kf, THR, KMAX) == 1
    assert_index(hb, eng, st.rows, what="after emptying")
    eng.close()


@pytest.mark.gpu
def test_changed_vector_threshold_or_kmax_rebuilds(hb):
    rng = np.random.default_rng(3)
    ta = rng.choice([-1.0, 1.0], DIM)
    rows = np.concatenate([_rows(rng, 900), _rows(rng, 150, ta)])
    eng = hb.Engine(0)
    assert eng.knn_index_update(rows, None, THR, KMAX) == 0
    changed = rows.copy()
    changed[500, 0] = -changed[500, 0]                     # a kept key's vector changed: detected, rebuilt
    assert eng.knn_index_update(changed, np.arange(rows.shape[0]), THR, KMAX) == 0
    assert_index(hb, eng, changed, what="changed vector")
    grown = np.concatenate([changed, _rows(rng, 50, ta)])
    grown[1000, 3] = -grown[1000, 3]                       # changed and appended in one call
    assert eng.knn_index_update(grown, np.arange(changed.shape[0]), THR, KMAX) == 0
    assert_index(hb, eng, grown, what="changed + append")
    n = grown.shape[0]
    assert eng.knn_index_update(grown, np.arange(n), 0.25, KMAX) == 0
    assert_index(hb, eng, grown, thr=0.25, what="threshold changed")
    assert eng.knn_index_update(grown, np.arange(n), 0.25, 40) == 0
    assert_index(hb, eng, grown, thr=0.25, kmax=40, what="kmax changed")
    assert eng.knn_index_update(grown, np.arange(n), 0.25, 40) == 2
    eng.close()


@pytest.mark.gpu
def test_rejected_calls_leave_the_index(hb):
    rng = np.random.default_rng(4)
    rows = _rows(rng, 700)
    eng = hb.Engine(0)
    eng.knn_index_update(rows, None, THR, KMAX)
    before = eng.knn_index_read()
    more = np.concatenate([rows, _rows(rng, 10)])
    bad = [dict(emb=more, kept_from=np.array([0, 2, 1])),                     # not increasing
           dict(emb=more, kept_from=np.array([0, 700])),                      # beyond the rows held
           dict(emb=more, kept_from=np.arange(-1, 5)),                        # negative
           dict(emb=rows[:, :60], kept_from=None),                            # dim % 8 != 0
           dict(emb=more, kept_from=np.arange(700), kmax=0),
           dict(emb=more, kept_from=np.arange(700), kmax=513),
           dict(emb=more, kept_from=np.arange(700), min_score=float("nan")),
           dict(emb=rows[:5], kept_from=np.arange(10))]                       # n_kept > rows
    for b in bad:
        with pytest.raises(hb.HragError):
            eng.knn_index_update(b["emb"], b["kept_from"], b.get("min_score", THR), b.get("kmax", KMAX))
        assert eng.knn_index_info() == (700, DIM, KMAX)
        after = eng.knn_index_read()
        assert np.array_equal(after[0], before[0]) and np.array_equal(after[1].view(np.uint32), before[1].view(np.uint32))
    eng.knn_index_clear()
    assert eng.knn_index_info() == (0, 0, 0)
    eng.close()


@pytest.mark.gpu
def test_resident_dict_equals_retrieve_knn(hb):
    """The ±1, d = 64 case of test_retrieve_knn_min_score_overflow_redo, served from the resident index after a build,
    a delete + append (ties across the old / new boundary) and with k < 128."""
    from hipporag_b200.knn import retrieve_knn, retrieve_knn_resident
    rng = np.random.default_rng(5)
    M = 1003
    keys = rng.choice([-1, 1], size=(M, DIM)).astype(np.float32)
    t = rng.choice([-1, 1], size=DIM).astype(np.float32)
    keys[rng.choice(M, 600, replace=False), :48] = t[:48]
    keys[11] = keys[3]
    ids = [f"k{i}" for i in range(M)]
    eng = hb.Engine(0)
    out, ran = retrieve_knn_resident(eng, ids, keys, 2047, 16 / 64, None)
    assert ran == "built" and out == retrieve_knn(ids, ids, keys, keys, k=2047, min_score=16 / 64)
    keep = np.ones(M, bool)
    keep[[0, 3, 500, 1002]] = False
    add = np.concatenate([keys[[11, 40]], rng.choice([-1, 1], size=(30, DIM)).astype(np.float32)])
    keys2 = np.concatenate([keys[keep], add])
    ids2 = [i for i, s in zip(ids, keep) if s] + [f"n{i}" for i in range(add.shape[0])]
    out, ran = retrieve_knn_resident(eng, ids2, keys2, 2047, 16 / 64, ids)
    assert ran == "updated" and out == retrieve_knn(ids2, ids2, keys2, keys2, k=2047, min_score=16 / 64)
    out, ran = retrieve_knn_resident(eng, ids2, keys2, 50, 16 / 64, ids2)
    assert ran == "built" and out == retrieve_knn(ids2, ids2, keys2, keys2, k=50, min_score=16 / 64)
    out, ran = retrieve_knn_resident(eng, ids2, keys2, 50, 16 / 64, ids2)
    assert ran == "unchanged"
    eng.close()


def _kg_engine(hb, kg, fe, pe):
    e = hb.Engine(0, mutable=True)
    e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    e.load_embeddings(fe, pe)
    return e


def _outputs(e, qf, qp, n_nodes):
    idx, score, nv = e.stage_a(qf, 5)
    ids, sc = e.stage_b(qp, idx, score, topk=50)
    ids2, sc2 = e.stage_b(qp[:4], idx[:4], score[:4], topk=50)
    pr = e.ppr(np.random.default_rng(1).random((3, n_nodes), dtype=np.float32))
    return [a.tobytes() for a in (idx, score, nv, ids, sc, ids2, sc2, pr)]


@pytest.mark.gpu
def test_retrieval_outputs_unaffected_by_the_knn_index(hb):
    from hipporag_b200 import synth
    kg = synth.make_kg(3000, 30000, seed=5)
    fe, pe = synth.unit_rows(kg.n_facts, DIM, 1), synth.unit_rows(kg.n_pass, DIM, 2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 40, seed=3)
    a, b = _kg_engine(hb, kg, fe, pe), _kg_engine(hb, kg, fe, pe)
    want = _outputs(a, qf, qp, kg.n_nodes)
    rng = np.random.default_rng(2)
    ents = _rows(rng, 2000)
    b.knn_index_update(ents, None, THR, KMAX)
    assert _outputs(b, qf, qp, kg.n_nodes) == want
    N = kg.n_nodes
    cc = np.r_[kg.ent_chunk_count, [1, 2, 0]].astype(np.int32)
    for e in (a, b):
        e.append(3, np.array([N, N + 1, 5], np.int32), np.array([7, 9, N + 2], np.int32), np.array([1.0, 0.5, 2.0]),
                 np.array([N + 2], np.int32), np.array([N, 3], np.int32), np.array([N + 1, -1], np.int32), cc,
                 fe[:2], pe[:1])
    b.knn_index_update(np.concatenate([ents, _rows(rng, 100)]), np.arange(2000), THR, KMAX)
    assert _outputs(b, qf, qp, N + 3) == _outputs(a, qf, qp, N + 3)
    for e in (a, b):
        e.delete(np.array([0, 11, N + 1], np.int32), np.array([1, 4], np.int32),
                 np.delete(cc, [0, 11, N + 1]).astype(np.int32))
    assert b.knn_index_info()[0] == 2100                   # the retrieval index's updates leave it alone
    assert _outputs(b, qf, qp, N) == _outputs(a, qf, qp, N)
    a.close()
    b.close()
