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

``retrieve_knn_resident`` serves the self-KNN (query ids == key ids) of the second form from an engine's resident index
(``hrag_knn_index_update``), which keeps the lists between calls and scores only the keys that changed, with the same
result; ``accelerate(incremental=True)`` routes ``add_synonymy_edges`` there.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

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


def classify_keys(old: Optional[Sequence[str]], new: Sequence[str]) -> Optional[np.ndarray]:
    """How the key list moved from ``old`` to ``new``: ``kept_from`` (int64), the positions in ``old`` of the first
    ``len(kept_from)`` keys of ``new``, when ``new`` is some of ``old``'s keys in their old order followed by keys
    ``old`` does not hold -- what ``EmbeddingStore`` insert (appends) and delete (compacts in order) produce.  ``None``
    (rebuild) for anything else: no old list, duplicates, a reorder, an old key after a new one."""
    if old is None:
        return None
    pos = {k: i for i, k in enumerate(old)}
    if len(pos) != len(old) or len(set(new)) != len(new):
        return None
    kept: List[int] = []
    for k in new:
        i = pos.get(k)
        if i is None:
            break
        if kept and i <= kept[-1]:
            return None
        kept.append(i)
    if any(k in pos for k in new[len(kept):]):
        return None
    return np.asarray(kept, dtype=np.int64)


def resident_exact(min_score: float) -> bool:
    """The resident index reproduces ``retrieve_knn(min_score=t)`` for thresholds float32 does not round down: the
    GEMM epilogue compares the float32 score with float32(t), while the overflow redo cuts in float64 at t itself, and
    the two agree on every float32 score only when float32(t) >= t (0.8, for one)."""
    return bool(np.isfinite(min_score)) and float(np.float32(min_score)) >= float(min_score)


def retrieve_knn_resident(engine: Engine, key_ids: Sequence[str], key_vecs, k: int, min_score: float,
                          prev_keys: Optional[Sequence[str]] = None) -> Tuple[Dict[str, Tuple[List[str], List[float]]],
                                                                               str]:
    """``retrieve_knn(key_ids, key_ids, key_vecs, key_vecs, k, min_score=min_score)`` served from ``engine``'s resident
    self-KNN index, which follows the change from ``prev_keys`` (the keys of the index's last update; ``None`` =
    unknown) in place: only the new keys are scored against the kept ones, only new and refilled rows against all.
    Returns (the same dict, bit for bit, "built" / "updated" / "unchanged").  Raises ``HragError`` when the library
    rejects the call (the index is then as it was, or cleared after a failure past validation)."""
    keys = _unit_rows(key_vecs)
    kept_from = classify_keys(prev_keys, list(key_ids))
    mode = engine.knn_index_update(keys, kept_from, float(min_score), int(min(k, MAX_CONSUMED)))
    ids, scores = engine.knn_index_read()
    return lists_to_dict(key_ids, ids, scores), ("built", "updated", "unchanged")[mode]


def lists_to_dict(key_ids: Sequence[str], ids: np.ndarray, scores: np.ndarray):
    """retrieve_knn's return value from [rows, kmax] id / score lists (-1 padded) of the keys against themselves."""
    out: Dict[str, Tuple[List[str], List[float]]] = {}
    for i, qid in enumerate(key_ids):
        n = int((ids[i] >= 0).sum())
        out[qid] = ([key_ids[j] for j in ids[i, :n]], scores[i, :n].tolist())
    return out
