"""Float64 CPU restatement of HippoRAG's online retrieval glue (SURVEY.md 8(a) rows
A-F) on integer tables.  TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

Every function cites the reference lines it follows (paths under
the reference's ``src/hipporag/``).  Differences from the reference, all deliberate:

* arithmetic is float64 from the same fp32 inputs (the reference's ``np.dot`` is an
  fp32 BLAS sgemv whose summation order no GPU kernel reproduces; float64 is the
  neutral arbiter, see SURVEY.md 7 hard part 3);
* ties are broken deterministically -- (score descending, index ascending) -- where
  the reference's outcome depends on ``np.argsort`` internals or Python ``set``
  iteration order (hard part 2);
* string keys (md5 of phrases) are replaced by vertex ids precomputed once, exactly
  the integer tables the engine uploads in ``prepare_retrieval_objects``.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import ppr as _ppr


def min_max_normalize(x: np.ndarray) -> np.ndarray:
    """``utils/misc_utils.py:130-139``: (x - min) / (max - min); all-equal -> ones."""
    x = np.asarray(x)
    lo, hi = x.min(), x.max()
    rng = hi - lo
    if rng == 0:
        return np.ones_like(x)
    return (x - lo) / rng


def order_desc(scores: np.ndarray, k: Optional[int] = None) -> np.ndarray:
    """Deterministic ranking: score descending, index ascending on ties."""
    scores = np.asarray(scores)
    idx = np.lexsort((np.arange(scores.shape[0]), -scores))
    return idx if k is None else idx[:k]


def fact_scores(fact_emb: np.ndarray, q_fact: np.ndarray) -> np.ndarray:
    """``HippoRAG.py:1427-1465``: s = E_f . q, min-max normalised; no facts -> empty."""
    if fact_emb.shape[0] == 0:
        return np.array([])
    s = fact_emb.astype(np.float64) @ q_fact.astype(np.float64)
    return min_max_normalize(s)


def top_facts(scores: np.ndarray, link_top_k: int) -> np.ndarray:
    """``HippoRAG.py:1683-1688``: indices of the ``linking_top_k`` best facts, best first."""
    if scores.shape[0] == 0:
        return np.zeros(0, dtype=np.int64)
    return order_desc(scores, min(link_top_k, scores.shape[0]))


def passage_scores(passage_emb: np.ndarray, q_pass: np.ndarray) -> np.ndarray:
    """``HippoRAG.py:1496-1498``: s = E_p . q, min-max normalised (unsorted; the sort at
    ``:1500`` is irrelevant to PPR and is re-derived by ``order_desc`` for DPR-only)."""
    s = passage_emb.astype(np.float64) @ q_pass.astype(np.float64)
    return min_max_normalize(s)


@dataclass
class Tables:
    """Integer tables equivalent to the dicts ``prepare_retrieval_objects`` builds
    (``HippoRAG.py:1287-1389``)."""
    n_nodes: int
    passage_vid: np.ndarray      # [P] vertex id of passage p  (passage_node_idxs, :1333)
    fact_subj_vid: np.ndarray    # [F] vertex id of the fact's subject entity, -1 if absent (:1591-1597)
    fact_obj_vid: np.ndarray     # [F] same for the object
    ent_chunk_count: np.ndarray  # [N] len(ent_node_to_chunk_ids[key]) (0 = absent) (:1598-1601)


def seed_vector(tables: Tables, fact_score_vec: np.ndarray, kept_fact_idx: Sequence[int],
                pass_scores_norm: np.ndarray, link_top_k: int = 5,
                passage_node_weight: float = 0.05):
    """Reset vector of ``graph_search_with_fact_entities`` (``HippoRAG.py:1577-1638``) and
    ``get_top_k_weights`` (``:1505-1542``).

    Returns (node_weights [N] float64, kept_phrase_vids).
    """
    N = tables.n_nodes
    phrase_w = np.zeros(N)
    occurs = np.zeros(N)
    touched = []
    for fidx in kept_fact_idx:                                   # :1583
        fs = float(fact_score_vec[fidx])                         # :1587-1588
        for vid in (int(tables.fact_subj_vid[fidx]), int(tables.fact_obj_vid[fidx])):  # :1590
            if vid < 0:                                          # :1597 (absent -> skipped)
                continue
            wfs = fs
            cnt = int(tables.ent_chunk_count[vid])
            if cnt > 0:                                          # :1600-1601
                wfs = fs / cnt
            phrase_w[vid] += wfs                                 # :1603
            occurs[vid] += 1                                     # :1604
            if vid not in touched:
                touched.append(vid)
    nz = occurs != 0
    phrase_w[nz] = phrase_w[nz] / occurs[nz]                     # :1608 (mean over occurrences)
    kept = list(touched)
    if link_top_k:                                               # :1620
        # :1528 keep the link_top_k best phrases; tie -> lower vertex id (documented policy)
        kept = sorted(touched, key=lambda v: (-phrase_w[v], v))[:link_top_k]
        mask = np.zeros(N, dtype=bool)
        mask[kept] = True
        phrase_w[~mask] = 0.0                                    # :1535-1539
    passage_w = np.zeros(N)
    # :1626-1633 ; the second min-max at :1627 is a numerical no-op (min 0, max 1)
    passage_w[tables.passage_vid] = pass_scores_norm * passage_node_weight
    return phrase_w + passage_w, kept                            # :1638


def retrieve_one(P_csr, tables: Tables, fact_emb, passage_emb, q_fact, q_pass,
                 link_top_k: int = 5, passage_node_weight: float = 0.05,
                 damping: float = 0.5, top_k: Optional[int] = None,
                 fact_filter=None, ppr_method: str = "power"):
    """One query through rows A-F (``HippoRAG.retrieve`` loop body, ``:459-480``).

    ``fact_filter(idx_list) -> idx_list`` stands in for the recognition-memory LLM
    filter (``:1696``); ``None`` is the identity filter used by every benchmark.
    Returns dict(ids, scores, facts, seeds, mode).
    """
    fs = fact_scores(fact_emb, q_fact)                           # row A
    cand = top_facts(fs, link_top_k)                             # row B
    kept = list(cand) if fact_filter is None else list(fact_filter(list(cand)))
    ps = passage_scores(passage_emb, q_pass)                     # row C
    if len(kept) == 0:                                           # :467-469 DPR fallback
        order = order_desc(ps, top_k)
        return dict(ids=order, scores=ps[order], facts=[], seeds=[], mode="dpr")
    r, phrases = seed_vector(tables, fs, kept, ps, link_top_k, passage_node_weight)  # row D
    if not r.sum() > 0:                                          # :1644
        raise AssertionError("No phrases found in the graph for the given facts")
    if ppr_method == "direct":
        pi = _ppr.ppr_direct(P_csr, r, damping)                  # row E
    else:
        pi = _ppr.ppr_power(P_csr, r, damping)
    doc = pi[tables.passage_vid]                                 # :1745
    order = order_desc(doc, top_k)                               # :1746 + slice :503
    return dict(ids=order, scores=doc[order], facts=kept, seeds=phrases, mode="ppr", reset=r)


def retrieve_batch(P_csr, tables: Tables, fact_emb, passage_emb, Q_fact, Q_pass, **kw):
    return [retrieve_one(P_csr, tables, fact_emb, passage_emb, Q_fact[i], Q_pass[i], **kw)
            for i in range(Q_fact.shape[0])]
