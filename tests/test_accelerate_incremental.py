"""accelerate(rag, incremental=True): index() / delete() followed in place on the device.

A test-local FakeRag whose index / delete mutate the fake igraph (add_vertices / add_edges / delete_vertices), the
stores and the embeddings the way the reference does (HippoRAG.py:262-335, :337-411).  Without a GPU, a recording
engine double checks the classification and that the recorded append / delete arguments, applied to the old
arrays, give extract_tables of the new state; on the GPU, retrieve after each update must equal a fresh incremental
load of the final state and match the default full reload.
"""
import numpy as np
import pytest

from tests import fake_hipporag

DIM = 64


def _key(prefix, name):
    from hipporag.utils.misc_utils import compute_mdhash_id
    return compute_mdhash_id(name, prefix)


class MutableRag(fake_hipporag.FakeRag):
    """FakeRag whose index()/delete() change the index.  index(spec): spec = dict(entities=[names], passages=[ids],
    edges=[(name_a, name_b, w)], facts=[(subj, obj)], chunks={entity: count}); delete(spec): spec = dict(
    passages=[ids], entities=[names], facts=[fact keys]).  Entity names are their content ("e12"), passage ids their
    number ("passage 12")."""

    def __init__(self, kg, fe, pe, qf, qp, queries):
        super().__init__(kg, fe, pe, qf, qp, queries)
        self._chunks = {self.entity_keys[v]: int(c) for v, c in enumerate(kg.ent_chunk_count[:kg.n_ent]) if c > 0}
        self._n_fact_keys = len(self.fact_node_keys)

    def prepare_retrieval_objects(self):
        self.node_name_to_vertex_idx = {n: i for i, n in enumerate(self.graph.vs["name"])}
        self.passage_node_idxs = [self.node_name_to_vertex_idx[k] for k in self.passage_node_keys]
        self.fact_embeddings, self.passage_embeddings = self._fact_emb, self._passage_emb
        self.ent_node_to_chunk_ids = {k: set(range(c)) for k, c in self._chunks.items()
                                      if k in self.node_name_to_vertex_idx}
        self.query_to_embedding = {"triple": {}, "passage": {}}
        self.ready_to_retrieve = True

    @staticmethod
    def _vertex(name):
        return _key("chunk-", name) if name.startswith("passage ") else _key("entity-", name)

    def index(self, spec):
        rng = np.random.default_rng(len(self.fact_node_keys))
        ents = [_key("entity-", e) for e in spec["entities"]]
        pks = [_key("chunk-", f"passage {i}") for i in spec["passages"]]
        self.graph.add_vertices(len(ents) + len(pks), attributes={"name": ents + pks})     # :1187
        self.graph.add_edges([(self._vertex(a), self._vertex(b)) for a, b, _ in spec["edges"]],
                             attributes={"weight": [w for _, _, w in spec["edges"]]})  # :1220
        for i, k in zip(spec["passages"], pks):
            self.chunk_embedding_store.rows[k] = {"hash_id": k, "content": f"passage {i}"}
        self.passage_node_keys = self.passage_node_keys + pks
        fkeys = []
        for s, o in spec["facts"]:
            k = f"fact-{self._n_fact_keys}"
            self._n_fact_keys += 1
            self.fact_embedding_store.rows[k] = {"hash_id": k, "content": str((s, "rel", o))}
            fkeys.append(k)
        self.fact_node_keys = self.fact_node_keys + fkeys
        self._fact_emb = np.concatenate([self._fact_emb, rng.standard_normal((len(fkeys), DIM)).astype(np.float32)])
        self._passage_emb = np.concatenate([self._passage_emb,
                                            rng.standard_normal((len(pks), DIM)).astype(np.float32)])
        self._chunks.update({_key("entity-", e): c for e, c in spec.get("chunks", {}).items()})

    def delete(self, spec):
        pks = [_key("chunk-", f"passage {i}") for i in spec["passages"]]
        ents = [_key("entity-", e) for e in spec["entities"]]
        self.graph.delete_vertices(pks + ents)                                              # :408
        kp = [k not in set(pks) for k in self.passage_node_keys]
        self.passage_node_keys = [k for k, s in zip(self.passage_node_keys, kp) if s]
        self._passage_emb = self._passage_emb[np.asarray(kp, bool)]
        kf = [k not in set(spec["facts"]) for k in self.fact_node_keys]
        self.fact_node_keys = [k for k, s in zip(self.fact_node_keys, kf) if s]
        self._fact_emb = self._fact_emb[np.asarray(kf, bool)]
        for e in ents:
            self._chunks.pop(e, None)
        self.ready_to_retrieve = False

    def reorder_facts(self):
        """A change no append or delete explains: the first two facts swap places."""
        self.fact_node_keys = [self.fact_node_keys[1], self.fact_node_keys[0]] + self.fact_node_keys[2:]
        self._fact_emb = self._fact_emb[np.r_[1, 0, 2:self._fact_emb.shape[0]]]
        self.ready_to_retrieve = False


def _make(seed=5):
    fake_hipporag.install_stub_package()
    from hipporag_b200 import synth
    kg = synth.make_kg(2000, 16000, seed=seed)
    fe, pe = synth.unit_rows(kg.n_facts, DIM, 1), synth.unit_rows(kg.n_pass, DIM, 2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 8, seed=3)
    return MutableRag(kg, fe, pe, qf, qp, [f"question {i}" for i in range(8)]), kg


def _ops(kg):
    """index -> delete -> index -> reorder, and what each must be classified as."""
    P = kg.n_pass
    add1 = dict(entities=[f"n{i}" for i in range(10)], passages=list(range(P, P + 5)),
                edges=[(f"passage {P + i % 5}", f"n{i}", 1.0) for i in range(8)]
                + [(f"passage {P + i}", f"e{3 * i + 1}", 1.0) for i in range(5)]
                + [("n0", "e5", 0.9), ("n0", "e5", 0.9), ("e1", "e2", 0.85), ("n3", "e9", 0.0)],
                facts=[("n0", "e5"), ("e5", "n0"), ("n1", "n3"), ("e2", "e40"), ("n4", "ghost")],
                chunks={"n0": 1, "n1": 2, "n3": 1, "n4": 1, "e5": 9})
    rm = dict(passages=[3, P + 1], entities=["n2", "e7"], facts=["fact-0", "fact-4"])
    add2 = dict(entities=["m0", "m1"], passages=[P + 5], edges=[(f"passage {P + 5}", "m0", 1.0), ("m1", "e11", 0.95)],
                facts=[("m0", "m1")], chunks={"m0": 1})
    return [("index", add1, "append"), ("delete", rm, "delete"), ("index", add2, "append"),
            ("reorder", None, "full")]


def _apply(rag, op, spec):
    if op == "index":
        rag.index(spec)
    elif op == "delete":
        rag.delete(spec)
    else:
        rag.reorder_facts()


# ----------------------------------------------------------------------------- CPU: classification, recorded calls
class RecordingEngine:
    """Engine double: keeps the arrays it was given and applies append / delete to them in numpy."""

    def __init__(self):
        self.calls, self.dim, self.mutable = [], 0, False

    def set_mutable(self, on=True):
        self.mutable = on

    def set_options(self, **kw):
        pass

    def load_graph(self, n, src, dst, w):
        self.calls.append("load_graph")
        self.n, self.src, self.dst, self.w = n, np.asarray(src, np.int32), np.asarray(dst, np.int32), np.asarray(w)

    def load_graph_csr(self, n, row_ptr, col, val):
        self.calls.append("load_graph_csr")

    def load_tables(self, pv, fs, fo, cc):
        self.calls.append("load_tables")
        self.pv, self.fs, self.fo, self.cc = (np.asarray(a, np.int32) for a in (pv, fs, fo, cc))

    def load_embeddings(self, fe, pe):
        self.calls.append("load_embeddings")
        self.fe, self.pe = np.asarray(fe, np.float32), np.asarray(pe, np.float32)
        self.dim = self.pe.shape[1]

    def append(self, n_new, src, dst, w, pv, fs, fo, cc, fe, pe):
        self.calls.append("append")
        assert self.mutable
        self.n += n_new
        self.src, self.dst, self.w = np.r_[self.src, src], np.r_[self.dst, dst], np.r_[self.w, w]
        self.pv, self.fs, self.fo, self.cc = np.r_[self.pv, pv], np.r_[self.fs, fs], np.r_[self.fo, fo], np.asarray(cc)
        self.fe, self.pe = np.concatenate([self.fe, fe]), np.concatenate([self.pe, pe])

    def delete(self, nodes, facts, cc):
        self.calls.append("delete")
        assert list(nodes) == sorted(set(nodes)) and list(facts) == sorted(set(facts))
        keep = np.ones(self.n, bool)
        keep[nodes] = False
        vmap = np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int32)
        ke, kp = keep[self.src] & keep[self.dst], keep[self.pv]
        kf = np.ones(self.fs.size, bool)
        kf[facts] = False
        rel = lambda v: np.where(v >= 0, vmap[np.maximum(v, 0)], -1).astype(np.int32)   # noqa: E731
        self.n = int(keep.sum())
        self.src, self.dst, self.w = vmap[self.src[ke]], vmap[self.dst[ke]], self.w[ke]
        self.pv, self.fs, self.fo, self.cc = vmap[self.pv[kp]], rel(self.fs[kf]), rel(self.fo[kf]), np.asarray(cc)
        self.fe, self.pe = self.fe[kf], self.pe[kp]


def _assert_engine_holds(eng, rag, state):
    from hipporag_b200.accelerate import extract_tables
    tb = extract_tables(rag)
    assert eng.n == tb["n_nodes"]
    for mine, theirs in ((eng.src, tb["edge_src"]), (eng.dst, tb["edge_dst"]), (eng.w, tb["edge_w"]),
                         (eng.pv, tb["passage_vid"]), (eng.fs, tb["fact_subj_vid"]), (eng.fo, tb["fact_obj_vid"]),
                         (eng.cc, tb["ent_chunk_count"]), (eng.fe, rag.fact_embeddings),
                         (eng.pe, rag.passage_embeddings)):
        assert np.asarray(mine).tobytes() == np.ascontiguousarray(theirs, dtype=np.asarray(mine).dtype).tobytes()
    assert state["facts"] == tb["facts"]


def test_incremental_classifies_and_records_what_extract_tables_gives():
    import hipporag_b200
    rag, kg = _make()
    eng = RecordingEngine()
    hipporag_b200.accelerate(rag, engine=eng, incremental=True, cache=False)
    rag.prepare_retrieval_objects()
    state = rag._b200_state
    assert state["last_update"] == "full" and eng.calls == ["load_graph", "load_tables", "load_embeddings"]
    _assert_engine_holds(eng, rag, state)
    for op, spec, want in _ops(kg):
        eng.calls.clear()
        _apply(rag, op, spec)
        rag.prepare_retrieval_objects()
        assert state["last_update"] == want, op
        assert eng.calls == ([want] if want != "full" else ["load_graph", "load_tables", "load_embeddings"])
        _assert_engine_holds(eng, rag, state)


def test_append_that_resolves_an_absent_fact_end_reloads():
    """A fact whose entity had no vertex keeps -1 in place; once an index() adds that entity, the row changes, so
    the update is a full reload."""
    import hipporag_b200
    rag, kg = _make()
    eng = RecordingEngine()
    hipporag_b200.accelerate(rag, engine=eng, incremental=True, cache=False)
    rag.prepare_retrieval_objects()
    rag.index(dict(entities=[], passages=[], edges=[], facts=[("e1", "later")]))
    rag.prepare_retrieval_objects()
    assert rag._b200_state["last_update"] == "append"
    rag.index(dict(entities=["later"], passages=[], edges=[("later", "e1", 1.0)], facts=[]))
    rag.prepare_retrieval_objects()
    assert rag._b200_state["last_update"] == "full"
    _assert_engine_holds(eng, rag, rag._b200_state)


def test_classify_update_fallbacks():
    from hipporag_b200.accelerate import classify_update
    old = dict(names=["a", "b", "c", "p"], edge_src=np.array([0, 1, 3], np.int32), edge_dst=np.array([1, 2, 0], np.int32),
               edge_w=np.array([1.0, 2.0, 3.0]), fact_keys=["f0", "f1"], passage_keys=["k0"],
               passage_vid=np.array([3], np.int32))

    def new(**kw):
        d = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in old.items()}
        d.update(kw)
        return d
    assert classify_update(old, new())[0] == "append"
    assert classify_update(old, new(names=["b", "a", "c", "p"]))[0] == "full"                 # reordered vertices
    assert classify_update(old, new(edge_w=np.array([1.0, 2.5, 3.0])))[0] == "full"          # a weight changed
    assert classify_update(old, new(fact_keys=["f1", "f0"]))[0] == "full"                    # reordered facts
    kind, info = classify_update(old, new(names=["a", "c", "p"], edge_src=np.array([2], np.int32),
                                          edge_dst=np.array([0], np.int32), edge_w=np.array([3.0]),
                                          fact_keys=["f1"], passage_vid=np.array([2], np.int32)))
    assert kind == "delete" and info["nodes"].tolist() == [1] and info["facts"].tolist() == [0]
    # the same delete with the surviving edges out of order, or a passage dropped whose vertex stayed
    assert classify_update(old, new(names=["a", "c", "p"], edge_src=np.array([0, 2], np.int32),
                                    edge_dst=np.array([0, 0], np.int32), edge_w=np.array([3.0, 3.0]),
                                    passage_vid=np.array([2], np.int32)))[0] == "full"
    assert classify_update(old, new(passage_keys=[], passage_vid=np.zeros(0, np.int32)))[0] == "full"


def test_default_mode_is_unchanged():
    """incremental=False: the host CSR is loaded, and every change reloads everything (no append / delete)."""
    import hipporag_b200
    rag, kg = _make()
    eng = RecordingEngine()
    hipporag_b200.accelerate(rag, engine=eng, cache=False)
    rag.prepare_retrieval_objects()
    for op, spec, _ in _ops(kg)[:2]:
        _apply(rag, op, spec)
        rag.prepare_retrieval_objects()
    assert eng.calls == ["load_graph_csr", "load_tables", "load_embeddings"] * 3
    assert not eng.mutable and "last_update" not in rag._b200_state


# ----------------------------------------------------------------------------- GPU: retrieve after the updates
@pytest.mark.gpu
def test_incremental_retrieve_equals_fresh_loads_on_gpu():
    import hipporag_b200
    from tests.util import assert_topk_matches
    rag, kg = _make()
    queries = [f"question {i}" for i in range(8)]
    hipporag_b200.accelerate(rag, device=0, incremental=True, cache=False)
    rag.retrieve(queries, num_to_retrieve=25)
    done = []
    for op, spec, want in _ops(kg):
        _apply(rag, op, spec)
        done.append((op, spec))
        got = rag.retrieve(queries, num_to_retrieve=25)
        assert rag._b200_state["last_update"] == want, op
        fresh, _ = _make()
        for o, s in done:
            _apply(fresh, o, s)
        hipporag_b200.accelerate(fresh, device=0, incremental=True, cache=False)
        want_sols = fresh.retrieve(queries, num_to_retrieve=25)
        for a, b in zip(got, want_sols):
            assert a.docs == b.docs and np.asarray(a.doc_scores).tobytes() == np.asarray(b.doc_scores).tobytes()
        full, _ = _make()
        for o, s in done:
            _apply(full, o, s)
        hipporag_b200.accelerate(full, device=0, cache=False)
        P = len(full.passage_node_keys)
        contents = [full.chunk_embedding_store.get_row(k)["content"] for k in full.passage_node_keys]
        index_of = {c: i for i, c in enumerate(contents)}
        for a, b in zip(got, full.retrieve(queries, num_to_retrieve=P)):
            o = np.zeros(P)
            o[[index_of[d] for d in b.docs]] = b.doc_scores
            assert_topk_matches([index_of[d] for d in a.docs], a.doc_scores, o, 25, what=op)
        for r in (fresh, full):
            r._b200_state["engine"].close()
