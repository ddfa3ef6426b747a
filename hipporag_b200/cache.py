"""Binary cache of what ``prepare_retrieval_objects`` has to rebuild for the engine (SURVEY.md 8(f)-3).

The reference persists the graph as ``<working_dir>/graph.pickle`` (``HippoRAG.py:225-233, 1229``) and the
embeddings as Parquet stores (``embedding_store.py:136-166``); every process start re-derives the retrieval
dicts from them in Python (``prepare_retrieval_objects`` ``:1287-1389``).  For the engine the expensive part
of that is ``accelerate.extract_tables``: one ``eval`` + two md5 lookups per fact and an edge-list walk --
O(F + E) Python.  This module stores its result next to ``graph.pickle``:

    <working_dir>/b200_index_cache.npz    CSR of P = W D^-1 (row_ptr int64, col int32, val float32), the integer
                                          tables (passage_vid, fact_subj_vid, fact_obj_vid, ent_chunk_count);
                                          with a float64 P also val_lo float32 = P - val (val + val_lo = P to
                                          ~2^-48 relative, the operator of ``accelerate(run_ppr_fp64=True)``)
    <working_dir>/b200_index_cache.json   fingerprint + the fact triples (the filter needs them as Python tuples)

keyed by a fingerprint of the index (vertex / edge / fact / passage counts, md5 of the vertex names, fact keys and
passage keys in order, md5 of the edge list and weights).  A changed index (``index()`` added documents,
``delete()``) changes the fingerprint and the cache is rebuilt: invalidation, not incremental patching.
The embedding matrices are not duplicated: their bf16 hi/lo planes are as large as the fp32 rows the Parquet
store already holds, and the device-side split takes milliseconds.
"""
from __future__ import annotations

import hashlib
import json
import os
from typing import Optional

import numpy as np

NPZ_NAME = "b200_index_cache.npz"
META_NAME = "b200_index_cache.json"
FORMAT_VERSION = 1


def _md5_of_strings(items) -> str:
    h = hashlib.md5()
    for s in items:
        h.update(str(s).encode("utf-8", "replace"))
        h.update(b"\0")
    return h.hexdigest()


def fingerprint(rag) -> dict:
    """Identity of the index state the cached arrays were derived from."""
    g = rag.graph
    edges = np.asarray(g.get_edgelist(), dtype=np.int64).reshape(-1, 2)
    weights = np.asarray(g.es["weight"], dtype=np.float64) if len(edges) else np.zeros(0)
    h = hashlib.md5()
    h.update(np.ascontiguousarray(edges).tobytes())
    h.update(np.ascontiguousarray(weights).tobytes())
    ent_chunks = rag.ent_node_to_chunk_ids or {}
    return {
        "format": FORMAT_VERSION,
        "n_nodes": int(g.vcount()), "n_edges": int(len(edges)),
        "n_facts": int(len(rag.fact_node_keys)), "n_passages": int(len(rag.passage_node_keys)),
        "vertex_names_md5": _md5_of_strings(g.vs["name"]) if g.vcount() else "",
        "fact_keys_md5": _md5_of_strings(rag.fact_node_keys),
        "passage_keys_md5": _md5_of_strings(rag.passage_node_keys),
        "edges_md5": h.hexdigest(),
        "chunk_counts_md5": _md5_of_strings(f"{k}:{len(v)}" for k, v in sorted(ent_chunks.items())),
    }


def save(working_dir: str, fp: dict, tables: dict, csr) -> None:
    """tables = accelerate.extract_tables(rag); csr = (row_ptr, col, val) of P.  A float64 ``val`` is stored as
    the float32 ``val`` plus ``val_lo``, so a float64 load (``load(..., fp64=True)``) gets P back to ~2^-48."""
    os.makedirs(working_dir, exist_ok=True)
    row_ptr, col, val = csr
    extra = {}
    if np.asarray(val).dtype == np.float64:
        hi = np.asarray(val, np.float32)
        extra["val_lo"] = (np.asarray(val, np.float64) - hi.astype(np.float64)).astype(np.float32)
    tmp = os.path.join(working_dir, NPZ_NAME + ".tmp.npz")
    np.savez(tmp, row_ptr=np.asarray(row_ptr, np.int64), col=np.asarray(col, np.int32), val=np.asarray(val, np.float32),
             passage_vid=np.asarray(tables["passage_vid"], np.int32),
             fact_subj_vid=np.asarray(tables["fact_subj_vid"], np.int32),
             fact_obj_vid=np.asarray(tables["fact_obj_vid"], np.int32),
             ent_chunk_count=np.asarray(tables["ent_chunk_count"], np.int32), **extra)
    os.replace(tmp, os.path.join(working_dir, NPZ_NAME))
    meta = {"fingerprint": fp, "facts": [list(f) for f in tables["facts"]]}
    tmpj = os.path.join(working_dir, META_NAME + ".tmp")
    with open(tmpj, "w") as f:
        json.dump(meta, f)
    os.replace(tmpj, os.path.join(working_dir, META_NAME))


def load(working_dir: str, fp: dict, fp64: bool = False) -> Optional[dict]:
    """The cached arrays if they were derived from exactly this index state, else None.  ``fp64``: ``val`` comes
    back as float64 ``val + val_lo``, and a cache without ``val_lo`` (written in the default mode) is a miss."""
    npz, meta = os.path.join(working_dir, NPZ_NAME), os.path.join(working_dir, META_NAME)
    if not (os.path.exists(npz) and os.path.exists(meta)):
        return None
    try:
        with open(meta) as f:
            m = json.load(f)
        if m.get("fingerprint") != fp:
            return None
        z = np.load(npz)
        out = {k: z[k] for k in ("row_ptr", "col", "val", "passage_vid", "fact_subj_vid", "fact_obj_vid",
                                 "ent_chunk_count")}
        if fp64:
            if "val_lo" not in z.files:
                return None
            out["val"] = out["val"].astype(np.float64) + z["val_lo"].astype(np.float64)
    except Exception:
        return None
    if out["row_ptr"].shape[0] != fp["n_nodes"] + 1 or out["fact_subj_vid"].shape[0] != fp["n_facts"]:
        return None
    out["n_nodes"] = fp["n_nodes"]
    out["facts"] = [tuple(f) for f in m["facts"]]
    return out
