"""accelerate(rag, incremental=True): the synonymy KNN of add_synonymy_edges served from the engine's resident index.

EntityRag keeps an entity store the way the reference's EmbeddingStore does (insert appends unseen keys, delete
compacts in order) and runs add_synonymy_edges' own walk of the KNN.  Without a GPU a recording engine checks the
key transitions it is given, the routing and the fallbacks; on the GPU the synonymy edges of index -> index -> delete
-> index equal those of incremental=False.
"""
import logging
import types

import numpy as np
import pytest

from tests import fake_hipporag

DIM = 64
retrieve_knn = fake_hipporag.retrieve_knn       # the module global add_synonymy_edges calls (HippoRAG.py:35)


class EntityStore:
    def __init__(self):
        self.keys, self.rows, self.emb = [], {}, np.zeros((0, DIM), np.float32)

    def insert(self, names, emb):
        new = [i for i, n in enumerate(names) if f"entity-{n}" not in self.rows]
        for i in new:
            k = f"entity-{names[i]}"
            self.keys.append(k)
            self.rows[k] = {"hash_id": k, "content": names[i]}
        self.emb = np.concatenate([self.emb, np.asarray(emb, np.float32)[new]])

    def delete(self, names):
        gone = {f"entity-{n}" for n in names}
        keep = np.array([k not in gone for k in self.keys], bool)
        self.keys = [k for k, s in zip(self.keys, keep) if s]
        self.emb = self.emb[keep]
        for k in gone:
            self.rows.pop(k, None)

    def get_all_id_to_rows(self):
        return {k: self.rows[k] for k in self.keys}

    def get_embeddings(self, keys):
        index = {k: i for i, k in enumerate(self.keys)}
        return self.emb[[index[k] for k in keys]]


class EntityRag:
    def __init__(self, thr=0.8, dim=DIM):
        self.global_config = types.SimpleNamespace(synonymy_edge_topk=2047, synonymy_edge_sim_threshold=thr,
                                                   synonymy_edge_query_batch_size=1000,
                                                   synonymy_edge_key_batch_size=10000)
        self.entity_embedding_store = EntityStore()
        self.node_to_node_stats = {}
        self.query_subset = None
        self.ready_to_retrieve = False

    def prepare_retrieval_objects(self):
        self.ready_to_retrieve = True

    def index(self, spec):
        names, emb = spec
        self.entity_embedding_store.insert(names, emb)
        self.add_synonymy_edges()

    def delete(self, names):
        self.entity_embedding_store.delete(names)

    def add_synonymy_edges(self):
        """HippoRAG.add_synonymy_edges' walk of the KNN (HippoRAG.py:980-1018)."""
        import re
        self.node_to_node_stats = {}
        rows = self.entity_embedding_store.get_all_id_to_rows()
        keys = list(rows.keys())
        embs = self.entity_embedding_store.get_embeddings(keys)
        qk = keys if self.query_subset is None else keys[:self.query_subset]
        qv = embs if self.query_subset is None else embs[:self.query_subset]
        knn = retrieve_knn(query_ids=qk, key_ids=keys, query_vecs=qv, key_vecs=embs,
                           k=self.global_config.synonymy_edge_topk)
        for node_key in knn.keys():
            if len(re.sub('[^A-Za-z0-9]', '', rows[node_key]["content"])) > 2:
                num_nns = 0
                for nn, score in zip(*knn[node_key]):
                    if score < self.global_config.synonymy_edge_sim_threshold or num_nns > 100:
                        break
                    if nn != node_key and rows[nn]["content"] != '':
                        self.node_to_node_stats[(node_key, nn)] = score
                        num_nns += 1


def _entities(rng, n, start, dim=DIM):
    """n named entities, +-1 rows in clusters sharing 60 of 64 coordinates (cosine >= 56/64 inside a cluster)."""
    t = rng.choice([-1.0, 1.0], size=(7, dim))
    x = rng.choice([-1.0, 1.0], size=(n, dim))
    c = rng.integers(0, 7, n)
    x[:, :dim - 4] = t[c, :dim - 4]
    x[c == 6] = rng.choice([-1.0, 1.0], size=(int((c == 6).sum()), dim))       # unclustered
    return [f"entity {start + i}" for i in range(n)], (x * rng.uniform(0.5, 2.0, (n, 1))).astype(np.float32)


def _ops(rng):
    a = _entities(rng, 300, 0)
    b = _entities(rng, 80, 300)
    c = _entities(rng, 50, 380)
    return [("index", a), ("index", b), ("delete", [f"entity {i}" for i in (0, 5, 17, 301, 333)]), ("index", c)]


def _run(rag, ops):
    for op, spec in ops:
        if op == "index":
            rag.index(spec)
        else:
            rag.delete(spec)


class RecordingEngine:
    """Engine double: records knn_index_update calls and serves the lists by an exact numpy all-pairs KNN."""

    def __init__(self, reject=0):
        self.calls, self.reject = [], reject
        self.keys = None

    def set_mutable(self, on=True):
        pass

    def knn_index_update(self, emb, kept_from, min_score, kmax):
        from hipporag_b200 import HragError
        if self.reject:
            self.reject -= 1
            raise HragError("rejected")
        self.calls.append((emb.shape[0], None if kept_from is None else np.asarray(kept_from).tolist()))
        unchanged = (self.keys is not None and kept_from is not None and emb.shape[0] == self.keys.shape[0]
                     and list(kept_from) == list(range(emb.shape[0])))
        self.keys = np.asarray(emb, np.float32)
        S = (self.keys @ self.keys.T).astype(np.float32)
        n = S.shape[0]
        self.ids = np.full((n, kmax), -1, np.int32)
        self.scores = np.zeros((n, kmax), np.float32)
        for r in range(n):
            order = np.lexsort((np.arange(n), -S[r]))
            order = order[S[r, order] >= np.float32(min_score)][:kmax]
            self.ids[r, :order.size], self.scores[r, :order.size] = order, S[r, order]
        return 2 if unchanged else (1 if kept_from is not None else 0)

    def knn_index_read(self):
        return self.ids, self.scores


def _accelerated(engine, thr=0.8, incremental=True, **kw):
    fake_hipporag.install_stub_package()
    import hipporag_b200
    rag = EntityRag(thr)
    hipporag_b200.accelerate(rag, engine=engine, incremental=incremental, cache=False, **kw)
    return rag


@pytest.fixture
def per_call(monkeypatch):
    """knn.retrieve_knn replaced by the numpy contract (the per-call path needs a GPU): records its calls."""
    from hipporag_b200 import knn
    calls = []

    def fake(query_ids, key_ids, query_vecs, key_vecs, k=2047, min_score=None, **kw):
        calls.append(len(key_ids))
        out = fake_hipporag.retrieve_knn(query_ids, key_ids, query_vecs, key_vecs, k=min(k, 128))
        return {q: ([i for i, s in zip(*v) if s >= min_score], [s for s in v[1] if s >= min_score])
                for q, v in out.items()}
    monkeypatch.setattr(knn, "retrieve_knn", fake)
    return calls


def test_routing_and_kept_from(per_call):
    eng = RecordingEngine()
    rag = _accelerated(eng)
    rng = np.random.default_rng(0)
    ops = _ops(rng)
    seen = []
    for op, spec in ops:
        _run(rag, [(op, spec)])
        if op == "index":
            seen.append(rag._b200_state["last_knn"])
    assert seen == ["built", "updated", "updated"] and per_call == []
    # build of 300; 300 kept + 80 new; (delete: no KNN call); 375 kept of 380 + 50 new
    assert [c[0] for c in eng.calls] == [300, 380, 425]
    assert eng.calls[0][1] is None and eng.calls[1][1] == list(range(300))
    gone = {0, 5, 17, 301, 333}
    assert eng.calls[2][1] == [i for i in range(380) if i not in gone]
    rag.add_synonymy_edges()                      # nothing changed
    assert rag._b200_state["last_knn"] == "unchanged" and eng.calls[-1][1] == list(range(425))
    # the edges are those of the plain KNN
    plain = EntityRag()
    _run(plain, ops)
    assert rag.node_to_node_stats == plain.node_to_node_stats and len(plain.node_to_node_stats) > 1000


@pytest.mark.parametrize("case", ["subset", "dim", "threshold", "not incremental"])
def test_fallbacks_to_per_call(per_call, case):
    eng = RecordingEngine()
    rag = _accelerated(eng, thr=0.7 if case == "threshold" else 0.8, incremental=case != "not incremental")
    rng = np.random.default_rng(1)
    names, emb = _entities(rng, 120, 0, dim=60 if case == "dim" else DIM)
    if case == "dim":
        rag.entity_embedding_store.emb = np.zeros((0, 60), np.float32)
    if case == "subset":
        rag.query_subset = 50
    rag.index((names, emb))
    assert eng.calls == [] and per_call == [120]
    assert rag._b200_state.get("last_knn", "per-call") == "per-call"


def test_rejected_call_warns_falls_back_and_rebuilds(per_call, caplog):
    eng = RecordingEngine(reject=1)
    rag = _accelerated(eng)
    rng = np.random.default_rng(2)
    a, b = _entities(rng, 100, 0), _entities(rng, 20, 100)
    with caplog.at_level(logging.WARNING, logger="hipporag_b200.accelerate"):
        rag.index(a)
    assert rag._b200_state["last_knn"] == "per-call" and per_call == [100]
    assert any("resident synonymy KNN failed" in r.message for r in caplog.records)
    rag.index(b)                                  # the next call builds: the index's key list is unknown
    assert rag._b200_state["last_knn"] == "built" and eng.calls == [(120, None)]


@pytest.mark.gpu
def test_incremental_synonymy_edges_equal_per_call_on_gpu():
    rng = np.random.default_rng(3)
    ops = _ops(rng)
    fake_hipporag.install_stub_package()
    import hipporag_b200
    results = {}
    for incremental in (False, True):
        rag = EntityRag()
        hipporag_b200.accelerate(rag, device=0, incremental=incremental, cache=False)
        ran = []
        for op, spec in ops:
            _run(rag, [(op, spec)])
            ran.append(rag._b200_state.get("last_knn"))
            results.setdefault(op + str(len(ran)), []).append(dict(rag.node_to_node_stats))
        if incremental:
            assert ran == ["built", "updated", "updated", "updated"]
        else:
            assert set(ran) == {"per-call"}
        rag._b200_state["engine"] and rag._b200_state["engine"].close()
    for step, (want, got) in results.items():
        assert got == want, step
    assert len(results["index4"][0]) > 1000
