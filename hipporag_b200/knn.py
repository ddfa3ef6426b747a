"""Index-time synonymy KNN on the H100 engine (SURVEY.md 8(f)-2).

Drop-in for ``hipporag.utils.embed_utils.retrieve_knn``
(reference ``src/hipporag/utils/embed_utils.py:6-94``, called from ``add_synonymy_edges``,
``HippoRAG.py:986-992``): cosine top-k of every query vector against all key vectors.  The reference
tiles ``torch.mm`` + ``torch.topk`` with CPU<->GPU ping-pong per tile; here the keys are uploaded once
and every query chunk is one wgmma GEMM.

Two forms:

* ``min_score=None`` -- the reference's contract as written: the full top-k (k <= 2048) per query
  (GEMM + exact radix top-k on the score chunk);
* ``min_score=t`` -- the contract as ``add_synonymy_edges`` *consumes* it (``HippoRAG.py:1003-1018``): the
  caller walks each neighbour list in score order and stops at the first score < ``synonymy_edge_sim_threshold``
  or once more than 100 neighbours were accepted, so only the entries >= t (and at most ~100 of them) can matter.
  The threshold is applied inside the GEMM epilogue (``hrag_knn_threshold``): no ``[chunk, N_ent]`` score
  matrix, no 2047-wide top-k.  ``accelerate()`` uses this form when it wraps ``add_synonymy_edges``.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

from .engine import Engine

# add_synonymy_edges accepts at most 101 neighbours per node (``num_nns > 100`` -> break) and skips only the node
# itself and empty phrases on the way: 128 entries always cover what it can read
MAX_CONSUMED = 128


def _unit_rows(x) -> np.ndarray:
    x = np.ascontiguousarray(x, dtype=np.float32)
    n = np.linalg.norm(x, axis=1, keepdims=True)
    return x / np.maximum(n, 1e-12)                     # torch.nn.functional.normalize(dim=1), eps 1e-12


def retrieve_knn(query_ids: List[str], key_ids: List[str], query_vecs, key_vecs, k: int = 2047,
                 query_batch_size: int = 1000, key_batch_size: int = 10000, device: int = 0,
                 engine: Optional[Engine] = None,
                 min_score: Optional[float] = None) -> Dict[str, Tuple[List[str], List[float]]]:
    """Same signature and return value as the reference (the two batch-size arguments are accepted and
    ignored: nothing is tiled through the host).  Ties are broken by lower key index.  With ``min_score`` the
    lists hold only the neighbours with score >= min_score (at most ``min(k, 128)``), which is all the caller
    of the reference ever reads."""
    if len(key_vecs) == 0:
        return {}
    keys = _unit_rows(key_vecs)
    queries = _unit_rows(query_vecs)
    if keys.shape[1] % 4:
        raise ValueError("embedding dim must be a multiple of 4")
    eng = engine or Engine(device)
    try:
        eng.load_embeddings(keys, keys[:1])
        out: Dict[str, Tuple[List[str], List[float]]] = {}
        if min_score is not None and keys.shape[1] % 8 == 0:
            kmax = int(min(k, MAX_CONSUMED))
            ids, scores, found = eng.knn_threshold(0, queries, float(min_score), kmax)
            redo = np.nonzero(found > 512)[0]            # a list overflowed its 512-entry buffer: exact path for it
            if redo.size:
                rid, rsc = eng.topk_similarity(0, queries[redo], int(min(kmax, keys.shape[0])))
                for j, qi in enumerate(redo):
                    keep = rsc[j] >= min_score
                    ids[qi], scores[qi] = -1, 0.0
                    ids[qi, :keep.sum()] = rid[j][keep]
                    scores[qi, :keep.sum()] = rsc[j][keep]
            for i, qid in enumerate(query_ids):
                n = int((ids[i] >= 0).sum())
                out[qid] = ([key_ids[j] for j in ids[i, :n]], scores[i, :n].tolist())
            return out
        kk = int(min(k, keys.shape[0], 2048))
        ids, scores = eng.topk_similarity(0, queries, kk)
        for i, qid in enumerate(query_ids):
            if min_score is not None:
                n = int((scores[i] >= min_score).sum())
                out[qid] = ([key_ids[j] for j in ids[i, :n]], scores[i, :n].tolist())
            else:
                out[qid] = ([key_ids[j] for j in ids[i]], scores[i].tolist())
        return out
    finally:
        if engine is None:
            eng.close()
