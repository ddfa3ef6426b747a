"""Drop-in: put a ``HippoRAG`` object's online retrieval path on the H100 engine.

    import hipporag_b200
    rag = HippoRAG(...); rag.index(docs)
    hipporag_b200.accelerate(rag, device=0)
    rag.retrieve(queries) / rag.rag_qa(queries)        # same signatures, same return types

What is rebound (all paths under the reference's ``src/hipporag/``):

* ``prepare_retrieval_objects`` (``HippoRAG.py:1287-1389``) -- the original runs, then the graph,
  the integer tables equivalent to its dicts, and the embeddings are uploaded once;
* ``retrieve_dpr`` (``:665-732``) -- batched dense passage retrieval (no PPR);
* ``retrieve_ircot`` (``:509-558``) -- step-synchronous: each reasoning round is one batched retrieve;
* ``retrieve`` (``:413-499``) -- batched: stage A for all queries -> the object's own
  ``rerank_filter`` per query, unchanged, on the host (the LLM call of ``rerank.py:108``) ->
  stage B for all queries (in float64 to PRPACK's 1e-10 with ``run_ppr_fp64=True``); timers ``ppr_time`` / ``rerank_time`` / ``all_retrieval_time`` and the
  optional Recall@k evaluation behave as in the reference;
* ``run_ppr`` (``:1709-1749``), ``dense_passage_retrieval`` (``:1467-1502``), ``get_fact_scores``
  (``:1427-1465``) -- single-call forms for code that uses them directly; ``run_ppr`` in float64 to PRPACK's
  1e-10 with ``run_ppr_fp64=True``;
* ``index`` / ``delete`` (``:262``, ``:337``) -- additionally invalidate the device state
  (``index`` forgets to clear ``ready_to_retrieve`` in the reference); with ``incremental=True`` the next prepare
  applies the change to the device in place when it is an append or an ordered delete;
* with ``attach=`` (a blob from ``share(owner_rag)`` in another process) ``prepare_retrieval_objects`` maps the
  owner's index on the same GPU instead of uploading one, and ``index`` / ``delete`` raise;
* ``add_synonymy_edges`` (``:959-1020``) -- runs unchanged, but the ``retrieve_knn`` it calls
  (``utils/embed_utils.py:6-94``, imported into ``HippoRAG.py:35``) is the engine's fused
  threshold KNN for the duration of the call (``hipporag_b200/knn.py``); with ``incremental=True`` the self-KNN stays
  on the device and each call scores only what changed.

``linking_top_k`` (``config_utils.py:184``) may be anything in [1, 32] (<= 8 is selected inside the GEMM
epilogue, larger values by an exact radix select); beyond 32 ``retrieve`` raises instead of clamping.

The engine never falls back to the CPU: if the CUDA library or an H100 is missing this raises.
"""
from __future__ import annotations

import json
import logging
import struct
import time
import types
from typing import Dict, List, Optional, Tuple

import numpy as np

from ._lib import HragError
from .engine import Engine

logger = logging.getLogger(__name__)
MAX_LINKING_TOP_K = 32          # kMaxKeptFacts of the library (csrc/kernels.h)
SHARE_MAGIC = b"hipporag_b200 share\n"
SHARE_VERSION = 1


def wrap_share_blob(fingerprint: dict, engine_blob: bytes) -> bytes:
    """The blob ``share`` returns: magic, a uint32 header length, a JSON header (``SHARE_VERSION`` and the index
    fingerprint of ``cache.fingerprint``), then the engine's ``export_index`` blob."""
    head = json.dumps({"version": SHARE_VERSION, "fingerprint": fingerprint}, sort_keys=True).encode()
    return SHARE_MAGIC + struct.pack("<I", len(head)) + head + bytes(engine_blob)


def unwrap_share_blob(blob: bytes) -> Tuple[dict, bytes]:
    """(fingerprint, engine blob) of a ``share`` blob; ValueError for anything else, another version or a
    truncated header."""
    blob = bytes(blob)
    n0 = len(SHARE_MAGIC)
    if blob[:n0] != SHARE_MAGIC or len(blob) < n0 + 4:
        raise ValueError("not a blob written by hipporag_b200.share()")
    (n,) = struct.unpack_from("<I", blob, n0)
    if len(blob) < n0 + 4 + n:
        raise ValueError("the share blob is truncated")
    head = json.loads(blob[n0 + 4:n0 + 4 + n])
    if head.get("version") != SHARE_VERSION:
        raise ValueError(f"share blob version {head.get('version')}, this package reads version {SHARE_VERSION}: "
                         "share and attach with the same build")
    return head["fingerprint"], blob[n0 + 4 + n:]


def share(rag) -> bytes:
    """Owner side of one index served to several worker processes on the same GPU: after ``accelerate(rag)`` and
    ``rag.prepare_retrieval_objects()``, export the engine's index (``Engine.export_index``) wrapped with the index
    fingerprint.  A worker passes the blob to ``accelerate(its_rag, attach=blob)``.  This process must outlive the
    workers.  From now on ``rag``'s engine rejects reloads: to change the index, have every worker detach
    (``rag._b200_state["engine"].detach()`` there), call ``unexport()`` on this engine, update, and share again."""
    state = getattr(rag, "_b200_state", None)
    if state is None or not state.get("uploaded") or state.get("engine") is None:
        raise HragError("share(): call accelerate(rag) and rag.prepare_retrieval_objects() first")
    from . import cache as _cache
    return wrap_share_blob(_cache.fingerprint(rag), state["engine"].export_index())


def extract_tables(rag) -> dict:
    """Integer tables equivalent to the dicts ``prepare_retrieval_objects`` builds."""
    from hipporag.utils.misc_utils import compute_mdhash_id
    n = rag.graph.vcount()
    name_to_vid = rag.node_name_to_vertex_idx
    edges = np.asarray(rag.graph.get_edgelist(), dtype=np.int32).reshape(-1, 2)
    weights = np.asarray(rag.graph.es["weight"], dtype=np.float64) if len(edges) else np.zeros(0)
    passage_vid = np.asarray(rag.passage_node_idxs, dtype=np.int32)                 # :1333
    F = len(rag.fact_node_keys)
    subj = np.full(F, -1, dtype=np.int32)
    obj = np.full(F, -1, dtype=np.int32)
    facts: List[tuple] = []
    if F:
        rows = rag.fact_embedding_store.get_rows(rag.fact_node_keys)
        for i, key in enumerate(rag.fact_node_keys):
            f = eval(rows[key]["content"])                                          # :1693
            facts.append(f)
            subj[i] = name_to_vid.get(compute_mdhash_id(f[0].lower(), prefix="entity-"), -1)   # :1584, :1591-1595
            obj[i] = name_to_vid.get(compute_mdhash_id(f[2].lower(), prefix="entity-"), -1)
    cnt = np.zeros(n, dtype=np.int32)
    for key, chunks in (rag.ent_node_to_chunk_ids or {}).items():                   # :1598-1601
        vid = name_to_vid.get(key)
        if vid is not None:
            cnt[vid] = len(chunks)
    return dict(n_nodes=n, edge_src=edges[:, 0], edge_dst=edges[:, 1], edge_w=weights, passage_vid=passage_vid,
                fact_subj_vid=subj, fact_obj_vid=obj, ent_chunk_count=cnt, facts=facts)


def index_view(rag) -> dict:
    """What the engine mirrors of ``rag``'s index that is cheap to read (no ``eval``, no md5): vertex names, the
    igraph edge list with its weights, fact keys, passage keys and passage vertices."""
    edges = np.asarray(rag.graph.get_edgelist(), dtype=np.int32).reshape(-1, 2)
    weights = np.asarray(rag.graph.es["weight"], dtype=np.float64) if len(edges) else np.zeros(0)
    return dict(names=list(rag.graph.vs["name"]) if rag.graph.vcount() else [],
                edge_src=np.ascontiguousarray(edges[:, 0]), edge_dst=np.ascontiguousarray(edges[:, 1]),
                edge_w=weights, fact_keys=list(rag.fact_node_keys), passage_keys=list(rag.passage_node_keys),
                passage_vid=np.asarray(rag.passage_node_idxs, dtype=np.int32))


def _same_bits(a, b) -> bool:
    return a.shape == b.shape and np.ascontiguousarray(a).tobytes() == np.ascontiguousarray(b).tobytes()


def _subsequence(old: list, new: list):
    """Positions in ``old`` of the items of ``new`` when ``new`` is ``old`` with some items removed in order, else
    None."""
    pos = {k: i for i, k in enumerate(old)}
    if len(pos) != len(old):
        return None
    idx = [pos.get(k, -1) for k in new]
    if any(i < 0 for i in idx) or any(b <= a for a, b in zip(idx, idx[1:])):
        return None
    return np.asarray(idx, dtype=np.int64)


def classify_update(old: dict, new: dict):
    """How the index moved from ``old`` to ``new`` (both ``index_view``s):

    * ``("append", {...})``: old names, edges with their weights, fact keys, passage keys and passage vertices are all
      prefixes of the new ones -- what ``HippoRAG.index()`` does (the stores append, igraph ``add_vertices`` /
      ``add_edges``);
    * ``("delete", {...})``: the new state is the old one with some vertices removed in order, the edge list is the
      old one filtered and relabelled, fact keys are an ordered subsequence and the passages are those whose vertex
      stayed -- what ``HippoRAG.delete()`` does (``delete_vertices`` compacts in order, the stores pop in place);
    * ``("full", None)``: anything else.
    """
    n0, n = len(old["names"]), len(new["names"])
    e0, f0, p0 = old["edge_src"].size, len(old["fact_keys"]), len(old["passage_keys"])
    if (n >= n0 and new["names"][:n0] == old["names"] and new["edge_src"].size >= e0
            and _same_bits(new["edge_src"][:e0], old["edge_src"]) and _same_bits(new["edge_dst"][:e0], old["edge_dst"])
            and _same_bits(new["edge_w"][:e0], old["edge_w"]) and new["fact_keys"][:f0] == old["fact_keys"]
            and new["passage_keys"][:p0] == old["passage_keys"]
            and _same_bits(new["passage_vid"][:p0], old["passage_vid"])):
        return "append", {"n_new_nodes": n - n0, "edges_from": e0, "facts_from": f0, "passages_from": p0}
    kept = _subsequence(old["names"], new["names"])
    kept_facts = _subsequence(old["fact_keys"], new["fact_keys"])
    if kept is None or kept_facts is None or n == 0:
        return "full", None
    keep = np.zeros(n0, bool)
    keep[kept] = True
    vmap = np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int32)
    ke = keep[old["edge_src"]] & keep[old["edge_dst"]]
    kp = keep[old["passage_vid"]]
    if not (_same_bits(vmap[old["edge_src"][ke]], new["edge_src"]) and _same_bits(vmap[old["edge_dst"][ke]],
                                                                                   new["edge_dst"])
            and _same_bits(old["edge_w"][ke], new["edge_w"])
            and [k for k, s in zip(old["passage_keys"], kp) if s] == new["passage_keys"]
            and _same_bits(vmap[old["passage_vid"][kp]], new["passage_vid"])):
        return "full", None
    kf = np.zeros(f0, bool)
    kf[kept_facts] = True
    return "delete", {"nodes": np.flatnonzero(~keep).astype(np.int32), "facts": np.flatnonzero(~kf).astype(np.int32),
                      "kept_facts": kept_facts}


def _fact_ends(facts, name_to_vid):
    """Subject / object vertex of each fact triple, -1 when absent (``HippoRAG.py:1584``, ``:1591-1595``)."""
    from hipporag.utils.misc_utils import compute_mdhash_id
    subj = np.array([name_to_vid.get(compute_mdhash_id(f[0].lower(), prefix="entity-"), -1) for f in facts], np.int32)
    obj = np.array([name_to_vid.get(compute_mdhash_id(f[2].lower(), prefix="entity-"), -1) for f in facts], np.int32)
    return subj, obj


def _chunk_counts(rag, n, name_to_vid) -> np.ndarray:
    cnt = np.zeros(n, dtype=np.int32)
    for key, chunks in (rag.ent_node_to_chunk_ids or {}).items():                   # :1598-1601
        vid = name_to_vid.get(key)
        if vid is not None:
            cnt[vid] = len(chunks)
    return cnt


def _resident_knn_applies(query_ids, key_ids, query_vecs, key_vecs, thr: float) -> bool:
    """Whether a ``retrieve_knn`` call is the self-KNN the resident index serves exactly: the same ids and vectors on
    both sides, a non-empty [rows, dim] matrix with dim % 8 == 0, a threshold float32 does not round down."""
    from . import knn
    if list(query_ids) != list(key_ids) or len(key_ids) == 0 or not knn.resident_exact(thr):
        return False
    shape = np.shape(key_vecs)
    if len(shape) != 2 or shape[0] != len(key_ids) or shape[1] % 8:
        return False
    return query_vecs is key_vecs or np.array_equal(np.asarray(query_vecs), np.asarray(key_vecs))


def accelerate(rag, device: int = 0, engine: Optional[Engine] = None, filter_workers: int = 1,
               filter_chunk: int = 256, ppr_tol: float = 0.0, cache: bool = True, run_ppr_fp64: bool = False,
               incremental: bool = False, fact_device_bytes: Optional[int] = None, attach: Optional[bytes] = None,
               knn_device_bytes: Optional[int] = None, fact_lo_on_host: bool = False, **engine_opts):
    """Rebinds the hot-path methods of ``rag`` (a reference ``HippoRAG`` instance) in place.

    ``filter_workers > 1`` (SURVEY.md 8(f)-1) runs the per-query recognition-memory filter calls (LLM HTTP
    requests, ``rerank.py:95``) in a thread pool AND pipelines them against the GPU: the queries go through stage
    A in chunks of ``filter_chunk``, a chunk's filter calls are submitted the moment its candidates are back, and
    stage A of the next chunk runs while they are in flight (ctypes releases the GIL inside the library).  The
    default 1 keeps the reference's serial order in the calling thread.  ``ppr_tol`` = relative L1 accuracy asked
    of every PPR vector (0 = the library default 1e-6; PRPACK's own target is 1e-10 in float64).
    ``cache`` (SURVEY.md 8(f)-3): keep the CSR of P and the integer tables as ``b200_index_cache.npz/.json`` next to
    the reference's ``graph.pickle`` and reuse them while the index fingerprint is unchanged (``hipporag_b200/cache.py``).
    ``run_ppr_fp64=True`` serves ``run_ppr`` (and so the reference's own ``graph_search_with_fact_entities``, which
    calls it) at PRPACK's accuracy: the float64 P is uploaded, and every call solves in float64 to ``ppr_tol``
    (0 = 1e-10) and returns float64 scores (``Engine.ppr_f64``).  ``retrieve`` -- and so ``rag_qa`` and
    ``retrieve_ircot``, which call it -- runs stage B the same way (``Engine.stage_b_f64``): the reset vector built
    in the reference's dtypes, float64 PPR to ``ppr_tol``, float64 ``doc_scores`` as the reference returns them.
    ``retrieve_dpr`` has no PPR and is the same in both modes.
    ``incremental=True`` follows ``index()`` / ``delete()`` in place instead of reloading: the graph is loaded from
    the igraph edge list on a mutable handle (``Engine(mutable=True)``; the tables still come from the cache or
    ``extract_tables``), and after the reference's own ``prepare_retrieval_objects`` has run, the change is
    classified (``classify_update``): an append goes through ``Engine.append`` and an ordered delete through
    ``Engine.delete``, with only the new facts ``eval``-ed; anything else is the full reload.
    ``rag._b200_state["last_update"]`` records which ran ("append", "delete" or "full").  The synonymy KNN of
    ``add_synonymy_edges`` is then kept on the engine as well (``knn.retrieve_knn_resident``): each call scores only
    the entities added since the last one against the others (and lists that lost a neighbour they need), with the
    same result as the per-call KNN; ``rag._b200_state["last_knn"]`` records what ran ("built", "updated",
    "unchanged" or "per-call").  Incremental updates do not
    write the binary cache: the next cold start rebuilds it, as after any change today.  The default
    (``incremental=False``) loads the host-built CSR and reloads everything after ``index()`` / ``delete()``.
    ``fact_device_bytes`` (``Engine.set_fact_memory``): device memory the fact planes may take; a fact matrix larger
    than that is kept in pinned host memory and streamed through the GPU by every stage-A call, with the same results.
    Stage A then streams the planes once per call, so ``filter_workers > 1`` streams them once per ``filter_chunk``
    queries: give it a large ``filter_chunk``.  Host planes cannot be updated in place: with ``incremental=True``
    every ``index()`` / ``delete()`` takes the full reload.
    ``fact_lo_on_host=True`` (``Engine.set_fact_placement``, needs ``fact_device_bytes``): over the budget only the lo
    fact plane goes to pinned host memory and the hi plane stays resident, so stage A runs the stage-A screen at
    about its resident cost and reads only the candidates' lo rows over PCIe, with the same results; the budget must
    hold the hi plane (rows x dim x 2 bytes) plus two 256-row lo slices.  Like host planes it cannot be updated in
    place: with ``incremental=True`` every ``index()`` / ``delete()`` takes the full reload.
    ``knn_device_bytes`` (``Engine.knn_set_memory``, needs ``incremental=True``: only the resident self-KNN index uses
    it): device memory the synonymy KNN index's planes may take; larger planes are kept in pinned host memory and
    streamed through the GPU by every update, with the same synonymy edges and ``last_knn`` values.
    ``attach`` (a blob from ``share(owner_rag)`` in a process on the same GPU): after the reference's own
    ``prepare_retrieval_objects`` has run, the index fingerprint is checked against the owner's (a mismatch raises)
    and the engine maps the owner's index read-only (``Engine.attach``) instead of uploading one; only the fact
    triples the filter needs are read on the host (from the cache, else ``extract_tables``).  ``index()`` /
    ``delete()`` then raise: the owner updates the index (see ``share``).  ``attach`` excludes ``incremental``,
    ``fact_device_bytes`` and ``fact_lo_on_host`` (ValueError).
    ``engine_opts`` go to ``Engine.set_options``.
    """
    from hipporag.utils.misc_utils import QuerySolution

    if attach is not None and (incremental or fact_device_bytes is not None or fact_lo_on_host):
        raise ValueError("accelerate(attach=...) serves another process's index read-only: it excludes "
                         "incremental=True, fact_device_bytes and fact_lo_on_host")
    if fact_lo_on_host and fact_device_bytes is None:
        raise ValueError("accelerate(fact_lo_on_host=True) places the fact planes under a device budget: give "
                         "fact_device_bytes as well")
    if knn_device_bytes is not None and not incremental:
        raise ValueError("accelerate(knn_device_bytes=...) bounds the resident synonymy KNN index, which only "
                         "incremental=True keeps")
    if knn_device_bytes is not None and int(knn_device_bytes) < 0:
        raise ValueError("accelerate(knn_device_bytes=...) must be >= 0 (0 = no limit)")
    shared = unwrap_share_blob(attach) if attach is not None else None     # (fingerprint, engine blob)

    state: Dict[str, object] = {"engine": engine, "facts": [], "uploaded": False}
    # calling accelerate() again on the same object re-wraps the REFERENCE's methods, not the previous wrappers
    if not hasattr(rag, "_b200_orig"):
        rag._b200_orig = {"prepare": rag.prepare_retrieval_objects, "index": rag.index, "delete": rag.delete,
                          "add_synonymy_edges": getattr(rag, "add_synonymy_edges", None)}
    orig_prepare = rag._b200_orig["prepare"]
    orig_index = rag._b200_orig["index"]
    orig_delete = rag._b200_orig["delete"]
    orig_add_synonymy_edges = rag._b200_orig["add_synonymy_edges"]

    def _engine() -> Engine:
        if state["engine"] is None:
            state["engine"] = Engine(device, mutable=incremental)
        elif incremental and not state.get("mutable_set"):
            state["engine"].set_mutable()
        state["mutable_set"] = incremental
        if fact_device_bytes is not None:     # before every load, which is what applies it
            state["engine"].set_fact_memory(fact_device_bytes)
            if fact_lo_on_host:
                state["engine"].set_fact_placement(True)
        if knn_device_bytes is not None:      # before every KNN index update, which is what applies it
            state["engine"].knn_set_memory(knn_device_bytes)
        return state["engine"]

    def _embeddings(self):
        fe = np.asarray(self.fact_embeddings, dtype=np.float32)
        pe = np.asarray(self.passage_embeddings, dtype=np.float32)
        return (fe.reshape(len(self.fact_node_keys), -1) if fe.size else np.zeros((0, pe.shape[1]), np.float32)), pe

    def _try_update(self, eng: Engine, view: dict) -> str:
        """Applies the change since the last load in place; returns what ran ("append" / "delete") or "full" when
        it has to be reloaded."""
        old = state.get("view")
        if old is None:
            return "full"
        kind, info = classify_update(old, view)
        name_to_vid = self.node_name_to_vertex_idx
        n = len(view["names"])
        if kind == "append":
            f0, p0, e0 = info["facts_from"], info["passages_from"], info["edges_from"]
            old_subj, old_obj = state["fact_ends"]
            absent = np.flatnonzero((old_subj < 0) | (old_obj < 0))
            if absent.size:   # an old fact's entity that has a vertex now would change its row: not an append
                s, o = _fact_ends([state["facts"][i] for i in absent], name_to_vid)
                if np.any(s != old_subj[absent]) or np.any(o != old_obj[absent]):
                    return "full"
            new_keys = view["fact_keys"][f0:]
            rows = self.fact_embedding_store.get_rows(new_keys) if new_keys else {}
            new_facts = [eval(rows[k]["content"]) for k in new_keys]                           # :1693
            subj, obj = _fact_ends(new_facts, name_to_vid)
            fe, pe = _embeddings(self)
            eng.append(info["n_new_nodes"], view["edge_src"][e0:], view["edge_dst"][e0:], view["edge_w"][e0:],
                       view["passage_vid"][p0:], subj, obj, _chunk_counts(self, n, name_to_vid), fe[f0:], pe[p0:])
            state["facts"] = list(state["facts"]) + new_facts
            state["fact_ends"] = (np.r_[old_subj, subj].astype(np.int32), np.r_[old_obj, obj].astype(np.int32))
            return "append"
        if kind == "delete":
            eng.delete(info["nodes"], info["facts"], _chunk_counts(self, n, name_to_vid))
            kept = info["kept_facts"]
            state["facts"] = [state["facts"][i] for i in kept]
            keep = np.ones(len(old["names"]), bool)
            keep[info["nodes"]] = False
            vmap = np.where(keep, np.cumsum(keep) - 1, -1).astype(np.int32)
            state["fact_ends"] = tuple(np.where(a[kept] >= 0, vmap[np.maximum(a[kept], 0)], -1).astype(np.int32)
                                       for a in state["fact_ends"])
            return "delete"
        return "full"

    def prepare_incremental(self):
        eng = _engine()
        view = index_view(self)
        try:
            kind = _try_update(self, eng, view)
        except HragError as e:                # rejected, or the index was dropped: reload it whole
            logger.warning(f"b200 in-place index update failed, reloading: {e}")
            kind = "full"
        if kind == "full":
            from . import cache as _cache
            wd = getattr(self, "working_dir", None) if cache else None
            tb = _cache.load(wd, _cache.fingerprint(self)) if wd else None
            state["cache_hit"] = tb is not None
            if tb is None:
                tb = extract_tables(self)
            eng.load_graph(len(view["names"]), view["edge_src"], view["edge_dst"], view["edge_w"])
            eng.load_tables(tb["passage_vid"], tb["fact_subj_vid"], tb["fact_obj_vid"], tb["ent_chunk_count"])
            eng.load_embeddings(*_embeddings(self))
            state["facts"] = tb["facts"]
            state["fact_ends"] = (np.asarray(tb["fact_subj_vid"], np.int32), np.asarray(tb["fact_obj_vid"], np.int32))
        if engine_opts:
            eng.set_options(**engine_opts)
        state["view"] = view
        state["last_update"] = kind
        state["uploaded"] = True

    def prepare_attached(self):
        from . import cache as _cache
        fp = _cache.fingerprint(self)
        if fp != shared[0]:
            raise HragError("accelerate(attach=...): this HippoRAG object's index differs from the one the owner "
                            "shared (index fingerprints differ); load the same index, or share it again")
        eng = _engine()
        if eng.share_info()["role"] != "attached":
            eng.attach(shared[1])
        wd = getattr(self, "working_dir", None) if cache else None
        tb = _cache.load(wd, fp) if wd else None
        state["cache_hit"] = tb is not None
        state["facts"] = (tb if tb is not None else extract_tables(self))["facts"]
        if engine_opts:
            eng.set_options(**engine_opts)
        state["uploaded"] = True

    def prepare_retrieval_objects(self):
        orig_prepare()
        if shared is not None:
            return prepare_attached(self)
        if incremental:
            return prepare_incremental(self)
        eng = _engine()
        from . import cache as _cache
        from .engine import build_transition_csr
        wd = getattr(self, "working_dir", None) if cache else None
        tb = fp = None
        if wd:
            fp = _cache.fingerprint(self)
            tb = _cache.load(wd, fp, fp64=True) if run_ppr_fp64 else _cache.load(wd, fp)
        state["cache_hit"] = tb is not None
        if tb is None:
            tb = extract_tables(self)
            if run_ppr_fp64:
                csr = build_transition_csr(tb["n_nodes"], tb["edge_src"], tb["edge_dst"], tb["edge_w"],
                                           dtype=np.float64)
            else:
                csr = build_transition_csr(tb["n_nodes"], tb["edge_src"], tb["edge_dst"], tb["edge_w"])
            tb["row_ptr"], tb["col"], tb["val"] = csr
            if wd:
                try:
                    _cache.save(wd, fp, tb, csr)
                except OSError as e:                      # a read-only index directory must not break retrieval
                    logger.warning(f"b200 index cache not written: {e}")
        eng.load_graph_csr(tb["n_nodes"], tb["row_ptr"], tb["col"], tb["val"])
        eng.load_tables(tb["passage_vid"], tb["fact_subj_vid"], tb["fact_obj_vid"], tb["ent_chunk_count"])
        fe = np.asarray(self.fact_embeddings, dtype=np.float32)
        pe = np.asarray(self.passage_embeddings, dtype=np.float32)
        eng.load_embeddings(fe.reshape(len(self.fact_node_keys), -1) if fe.size else np.zeros((0, pe.shape[1]), np.float32), pe)
        if engine_opts:
            eng.set_options(**engine_opts)
        state["facts"] = tb["facts"]
        state["uploaded"] = True

    def _ensure_ready(self):
        if not self.ready_to_retrieve or not state["uploaded"]:
            self.prepare_retrieval_objects()

    def _query_matrix(self, queries: List[str], kind: str) -> np.ndarray:
        rows = []
        for q in queries:
            v = np.asarray(self.query_to_embedding[kind][q], dtype=np.float32)
            rows.append(v.reshape(-1))
        return np.stack(rows) if rows else np.zeros((0, _engine().dim), np.float32)

    def retrieve(self, queries: List[str], num_to_retrieve: int = None, gold_docs: List[List[str]] = None):
        retrieve_start_time = time.time()
        if num_to_retrieve is None:
            num_to_retrieve = self.global_config.retrieval_top_k
        if gold_docs is not None:
            from hipporag.evaluation.retrieval_eval import RetrievalRecall
            retrieval_recall_evaluator = RetrievalRecall(global_config=self.global_config)
        _ensure_ready(self)
        self.get_query_embeddings(queries)
        eng = _engine()
        link_top_k = self.global_config.linking_top_k
        facts_all = state["facts"]

        # ---- stage A on the GPU, then the recognition-memory filter on the host (unchanged)
        rerank_start = time.time()
        if not isinstance(link_top_k, (int, np.integer)) or link_top_k < 1:
            raise ValueError(f"linking_top_k must be a positive integer, got {link_top_k!r}")
        if link_top_k > MAX_LINKING_TOP_K:
            raise ValueError(f"linking_top_k = {link_top_k} exceeds the {MAX_LINKING_TOP_K} candidate facts per query "
                             "the engine keeps (it does not clamp silently)")
        k = int(link_top_k)
        nq = len(queries)
        Qf = _query_matrix(self, queries, "triple")
        idx = np.full((nq, k), -1, np.int32)
        score = np.zeros((nq, k), np.float32)
        nv = np.zeros(nq, np.int32)
        kept_idx = np.full((nq, k), -1, dtype=np.int32)
        kept_score = np.zeros((nq, k), dtype=np.float32)
        kept_facts: List[List[tuple]] = []

        def _filter_one(qi):
            cand_idx = [int(i) for i in idx[qi, :nv[qi]]]
            if not cand_idx:
                return cand_idx, [], []
            cand_facts = [facts_all[i] for i in cand_idx]
            try:
                top_idx, top_facts, _ = self.rerank_filter(queries[qi], cand_facts, cand_idx,
                                                           len_after_rerank=link_top_k)          # :1696-1699
            except Exception as e:                                                               # :1705-1707
                logger.error(f"Error in rerank_facts: {e}")
                top_idx, top_facts = [], []
            return cand_idx, top_idx, top_facts

        def _stage_a(lo, hi):
            if len(facts_all) and hi > lo:
                idx[lo:hi], score[lo:hi], nv[lo:hi] = eng.stage_a(Qf[lo:hi], k)

        if filter_workers > 1 and nq > 1:
            # pipelined: chunk c's filter calls run in the pool while the GPU scores chunk c + 1
            from concurrent.futures import ThreadPoolExecutor
            step = max(1, int(filter_chunk))
            futures = []
            with ThreadPoolExecutor(max_workers=filter_workers) as pool:
                for lo in range(0, nq, step):
                    hi = min(nq, lo + step)
                    _stage_a(lo, hi)
                    futures.extend(pool.submit(_filter_one, qi) for qi in range(lo, hi))
                filtered = [f.result() for f in futures]
        else:
            _stage_a(0, nq)
            filtered = [_filter_one(qi) for qi in range(nq)]
        for qi, (cand_idx, top_idx, top_facts) in enumerate(filtered):
            score_of = {i: float(s) for i, s in zip(cand_idx, score[qi, :nv[qi]])}
            top_idx = [int(i) for i in top_idx][:k]
            kept_idx[qi, :len(top_idx)] = top_idx
            kept_score[qi, :len(top_idx)] = [score_of.get(i, 0.0) for i in top_idx]
            kept_facts.append(list(top_facts)[:k])
        self.rerank_time += time.time() - rerank_start

        # ---- stage B on the GPU (DPR fallback per query where nothing was kept, :467-469)
        ppr_start = time.time()
        topk = int(min(num_to_retrieve, 2048, max(len(self.passage_node_keys), 1)))
        stage_b = eng.stage_b_f64 if run_ppr_fp64 else eng.stage_b
        ids, scores = stage_b(_query_matrix(self, queries, "passage"), kept_idx, kept_score, None,
                              self.global_config.damping, self.global_config.passage_node_weight,
                              link_top_k, topk, tol=ppr_tol)
        self.ppr_time += time.time() - ppr_start

        retrieval_results = []
        for qi, query in enumerate(queries):
            valid = ids[qi] >= 0
            result = self._build_retrieval_result(query, ids[qi][valid].astype(np.int64),
                                                  scores[qi][valid].astype(np.float64), num_to_retrieve,
                                                  kept_facts[qi])                                 # :478, :501-507
            retrieval_results.append(QuerySolution(question=result.query, docs=result.docs,
                                                   doc_scores=result.scores, doc_metadata=result.doc_metadata,
                                                   graph_seeds=result.graph_seeds))
        self.all_retrieval_time += time.time() - retrieve_start_time
        logger.info(f"Total Retrieval Time {self.all_retrieval_time:.2f}s")                        # :486-489
        logger.info(f"Total Recognition Memory Time {self.rerank_time:.2f}s")
        logger.info(f"Total PPR Time {self.ppr_time:.2f}s")
        logger.info(f"Total Misc Time {self.all_retrieval_time - (self.rerank_time + self.ppr_time):.2f}s")
        if gold_docs is not None:
            k_list = [1, 2, 5, 10, 20, 30, 50, 100, 150, 200]
            overall, _ = retrieval_recall_evaluator.calculate_metric_scores(
                gold_docs=gold_docs, retrieved_docs=[r.docs for r in retrieval_results], k_list=k_list)
            logger.info(f"Evaluation results for retrieval: {overall}")
            return retrieval_results, overall
        return retrieval_results

    def retrieve_dpr(self, queries: List[str], num_to_retrieve: int = None, gold_docs: List[List[str]] = None):
        """``HippoRAG.py:665-732``: dense passage retrieval only, batched on the GPU."""
        retrieve_start_time = time.time()
        if num_to_retrieve is None:
            num_to_retrieve = self.global_config.retrieval_top_k
        _ensure_ready(self)
        self.get_query_embeddings(queries)
        topk = int(min(num_to_retrieve, 2048, max(len(self.passage_node_keys), 1)))
        none_i = np.zeros((len(queries), 0), dtype=np.int32)
        ids, scores = _engine().stage_b(_query_matrix(self, queries, "passage"), none_i, none_i.astype(np.float32),
                                        None, self.global_config.damping, self.global_config.passage_node_weight,
                                        self.global_config.linking_top_k, topk)
        results = []
        for qi, query in enumerate(queries):
            valid = ids[qi] >= 0
            r = self._build_retrieval_result(query, ids[qi][valid].astype(np.int64),
                                             scores[qi][valid].astype(np.float64), num_to_retrieve)
            results.append(QuerySolution(question=r.query, docs=r.docs, doc_scores=r.scores,
                                         doc_metadata=r.doc_metadata, graph_seeds=r.graph_seeds))
        self.all_retrieval_time += time.time() - retrieve_start_time
        if gold_docs is not None:
            from hipporag.evaluation.retrieval_eval import RetrievalRecall
            overall, _ = RetrievalRecall(global_config=self.global_config).calculate_metric_scores(
                gold_docs=gold_docs, retrieved_docs=[r.docs for r in results],
                k_list=[1, 2, 5, 10, 20, 30, 50, 100, 150, 200])
            return results, overall
        return results

    def retrieve_ircot(self, queries: List[str], max_qa_steps: int, num_to_retrieve: int = None,
                       gold_docs: List[List[str]] = None):
        """``HippoRAG.py:509-558`` step-synchronously (SURVEY.md 8(f)-4): the reference runs, per query,
        retrieve([query]) then up to max_qa_steps-1 rounds of reason_step -> retrieve([thought]); queries
        are independent, so every round's retrievals are issued as ONE batched retrieve() over the
        queries still active.  Same merge rule (max score per document) and the same result objects."""
        from hipporag.utils.qa_utils import reason_step
        if max_qa_steps < 1:
            raise ValueError("max_qa_steps must be at least 1.")
        if num_to_retrieve is None:
            num_to_retrieve = self.global_config.retrieval_top_k
        prompt_name = f'ircot_{self.global_config.dataset}'
        if max_qa_steps > 1 and not self.prompt_template_manager.is_template_name_valid(prompt_name):
            raise ValueError(f"IRCoT prompt template '{prompt_name}' is not available.")
        first = self.retrieve(list(queries), num_to_retrieve=num_to_retrieve)
        merged_scores = [dict(zip(r.docs, np.asarray(r.doc_scores).tolist())) for r in first]
        merged_meta = [dict(zip(r.docs, r.doc_metadata or [])) for r in first]
        thoughts: List[List[str]] = [[] for _ in queries]
        active = list(range(len(queries)))
        for _ in range(1, max_qa_steps):
            if not active:
                break
            step_queries, step_owner = [], []
            for qi in active:
                ranked = sorted(merged_scores[qi], key=merged_scores[qi].get, reverse=True)
                thought = reason_step(self.global_config.dataset, self.prompt_template_manager, queries[qi],
                                      ranked[:num_to_retrieve], thoughts[qi], self.qa_llm)        # :533-534
                thoughts[qi].append(thought)
                if 'So the answer is:' in thought:                                                # :536
                    continue
                step_queries.append(thought)
                step_owner.append(qi)
            active = step_owner
            if not step_queries:
                break
            for qi, res in zip(step_owner, self.retrieve(step_queries, num_to_retrieve=num_to_retrieve)):
                for doc, score in zip(res.docs, np.asarray(res.doc_scores).tolist()):             # :540-541
                    merged_scores[qi][doc] = max(merged_scores[qi].get(doc, float('-inf')), score)
                merged_meta[qi].update(dict(zip(res.docs, res.doc_metadata or [])))
        results = []
        for qi, query in enumerate(queries):
            items = sorted(merged_scores[qi].items(), key=lambda it: it[1], reverse=True)
            results.append(QuerySolution(question=query, docs=[d for d, _ in items],
                                         doc_scores=np.asarray([sc for _, sc in items]), thoughts=thoughts[qi],
                                         doc_metadata=[merged_meta[qi].get(d, {}) for d, _ in items]))
        if gold_docs is None:
            return results
        from hipporag.evaluation.retrieval_eval import RetrievalRecall
        overall, _ = RetrievalRecall(global_config=self.global_config).calculate_metric_scores(
            gold_docs=gold_docs, retrieved_docs=[r.docs for r in results],
            k_list=[1, 2, 5, 10, 20, 30, 50, 100, 150, 200])
        return results, overall

    def run_ppr(self, reset_prob: np.ndarray, damping: float = 0.5) -> Tuple[np.ndarray, np.ndarray]:
        """``HippoRAG.py:1709-1749``; full-length ranking as the reference returns."""
        if damping is None:
            damping = 0.5
        _ensure_ready(self)
        if run_ppr_fp64:
            pi = _engine().ppr_f64(np.asarray(reset_prob, dtype=np.float64), damping, tol=ppr_tol)
        else:
            pi = _engine().ppr(np.asarray(reset_prob, dtype=np.float32), damping, tol=ppr_tol)
        doc_scores = pi[np.asarray(self.passage_node_idxs, dtype=np.int64)].astype(np.float64)
        order = np.lexsort((np.arange(doc_scores.shape[0]), -doc_scores))
        return order, doc_scores[order]

    def get_fact_scores(self, query: str) -> np.ndarray:
        _ensure_ready(self)
        if len(self.fact_node_keys) == 0:
            return np.array([])                                                                  # :1454-1456
        self.get_query_embeddings([query])
        return _engine().similarity(0, _query_matrix(self, [query], "triple"))[0]

    def dense_passage_retrieval(self, query: str) -> Tuple[np.ndarray, np.ndarray]:
        _ensure_ready(self)
        self.get_query_embeddings([query])
        s = _engine().similarity(1, _query_matrix(self, [query], "passage"))[0]
        order = np.lexsort((np.arange(s.shape[0]), -s))
        return order, s[order]

    def _reject_update(what):
        if shared is not None:
            raise HragError(f"{what}: this HippoRAG object serves an index attached from another process "
                            "(accelerate(attach=...)), which it only reads; update the index in the owner process "
                            "(see hipporag_b200.share)")

    def index(self, docs):
        _reject_update("index()")
        state["uploaded"] = False
        self.ready_to_retrieve = False
        return orig_index(docs)

    def delete(self, docs_to_delete):
        _reject_update("delete()")
        state["uploaded"] = False
        return orig_delete(docs_to_delete)

    def add_synonymy_edges(self):
        """``HippoRAG.py:959-1020`` unchanged, with the KNN it calls (``:986-992``) served by the engine: cosine
        >= synonymy_edge_sim_threshold selected inside the GEMM epilogue, no [chunk, N_ent] score matrix.  With
        ``incremental=True`` the self-KNN is served from the engine's resident index, updated in place; other calls
        (query ids != key ids, dim % 8 != 0, a threshold float32 rounds down, a rejected call) run per call."""
        import sys
        from . import knn
        mod = sys.modules[type(self).__module__]
        saved = getattr(mod, "retrieve_knn", None)
        thr = float(self.global_config.synonymy_edge_sim_threshold)

        def fused_knn(query_ids, key_ids, query_vecs, key_vecs, k=2047, query_batch_size=1000, key_batch_size=10000):
            if incremental and _resident_knn_applies(query_ids, key_ids, query_vecs, key_vecs, thr):
                try:
                    out, ran = knn.retrieve_knn_resident(_engine(), key_ids, key_vecs, k, thr, state.get("knn_keys"))
                    state["knn_keys"], state["last_knn"] = list(key_ids), ran
                    return out
                except HragError as e:           # rejected (or the index was dropped): today's per-call path
                    logger.warning(f"b200 resident synonymy KNN failed, running it per call: {e}")
                    state["knn_keys"] = None
            state["last_knn"] = "per-call"
            return knn.retrieve_knn(query_ids, key_ids, query_vecs, key_vecs, k=k, query_batch_size=query_batch_size,
                                    key_batch_size=key_batch_size, device=device, min_score=thr)
        mod.retrieve_knn = fused_knn
        try:
            return orig_add_synonymy_edges()
        finally:
            if saved is not None:
                mod.retrieve_knn = saved

    for name, fn in (("prepare_retrieval_objects", prepare_retrieval_objects), ("retrieve", retrieve),
                     ("retrieve_dpr", retrieve_dpr), ("retrieve_ircot", retrieve_ircot),
                     ("run_ppr", run_ppr), ("get_fact_scores", get_fact_scores),
                     ("dense_passage_retrieval", dense_passage_retrieval), ("index", index), ("delete", delete)):
        setattr(rag, name, types.MethodType(fn, rag))
    if orig_add_synonymy_edges is not None:
        setattr(rag, "add_synonymy_edges", types.MethodType(add_synonymy_edges, rag))
    rag._b200_state = state
    return rag
