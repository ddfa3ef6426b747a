"""Seeded synthetic knowledge graphs of the shapes BASELINE.json names (SURVEY.md 8(d)).

There is no network for datasets, so configs C2-C5 are generated: a knowledge graph with
the edge mix the reference's ``index()`` produces on MuSiQue
(reference ``src/hipporag/HippoRAG.py:867-957,959-1020``):

* ~55 % of the igraph edges are *fact* edges, emitted as PAIRS of parallel edges (s,o) and
  (o,s), each carrying the co-occurrence count (``:907-910``);
* ~35 % passage->entity edges of weight 1.0 (``:953``);
* ~10 % synonymy edges with weight U[0.8, 1.0) (``:1007-1018``);
* vertex order: entities first, then passages (``:1174-1175``); 0.1 % of the entities are
  left isolated so sinks are exercised.

Everything is numpy on the host and deterministic in ``seed``.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np


@dataclass
class SynthKG:
    n_nodes: int
    n_ent: int
    n_pass: int
    edge_src: np.ndarray         # [E] int32   igraph-style undirected multigraph edge list
    edge_dst: np.ndarray         # [E] int32
    edge_w: np.ndarray           # [E] float64
    passage_vid: np.ndarray      # [P] int32   vertex id of passage p
    fact_subj_vid: np.ndarray    # [F] int32
    fact_obj_vid: np.ndarray     # [F] int32
    ent_chunk_count: np.ndarray  # [N] int32   #passages containing the entity (0 for passages)
    fact_passage: np.ndarray     # [F] int32   a passage adjacent to the fact's subject (query planting)

    @property
    def n_facts(self):
        return int(self.fact_subj_vid.shape[0])

    @property
    def n_edges(self):
        return int(self.edge_src.shape[0])


def make_kg(n_nodes: int, n_edges: int, seed: int = 0, topology: str = "uniform",
            zipf_s: float = 1.1, zipf_q: float = None) -> SynthKG:
    """Graph with ``n_nodes`` vertices (90 % entities, 10 % passages) and ~``n_edges`` igraph edges.

    ``topology="powerlaw"`` (BASELINE config #5): entity endpoints follow a shifted Zipf law
    p(rank) ~ (rank + zipf_q)^-zipf_s, zipf_q defaulting to 150 per 9M entities.  With s = 1.1 the heaviest
    entity of the 10M-node graph then collects ~1e-3 of all endpoints -- a hub of degree ~1e5 as SURVEY.md 8(d)
    asks -- where the unshifted law (q = 0) would put 6 % of all endpoints on one vertex and lose a third of the
    edges to duplicates."""
    rng = np.random.default_rng(seed)
    n_pass = max(1, n_nodes // 10)
    n_ent = n_nodes - n_pass
    n_iso = max(1, n_ent // 1000) if n_ent >= 100 else 0
    n_live = n_ent - n_iso                      # isolated entities are the last n_iso entity ids

    def draw_entities(k):
        if topology == "uniform":
            return rng.integers(0, n_live, size=k, dtype=np.int64)
        if topology == "powerlaw":
            # Zipf(s) over entity ranks through the inverse CDF of the continuous analogue
            u = rng.random(k)
            q = float(zipf_q) if zipf_q is not None else 150.0 * n_live / 9.0e6
            if abs(zipf_s - 1.0) < 1e-9:
                r = (1.0 + q) * np.exp(u * np.log((n_live + q) / (1.0 + q))) - q
            else:
                a = 1.0 - zipf_s
                lo, hi = (1.0 + q) ** a, (n_live + q) ** a
                r = (lo + u * (hi - lo)) ** (1.0 / a) - q
            return np.minimum(r.astype(np.int64) - 1, n_live - 1).clip(0)
        raise ValueError(topology)

    n_fact_pairs = int(round(0.275 * n_edges))
    n_pe = int(round(0.35 * n_edges))
    n_syn = n_edges - 2 * n_fact_pairs - n_pe

    # facts: distinct (subject, object) entity pairs, s != o
    over = 1.15 if topology == "uniform" else 1.35      # duplicates are commoner among Zipf draws
    s = draw_entities(int(n_fact_pairs * over) + 16)
    o = draw_entities(s.shape[0])
    ok = s != o
    s, o = s[ok], o[ok]
    key = np.unique(s * n_ent + o)
    rng.shuffle(key)
    key = key[:n_fact_pairs]
    fs, fo = (key // n_ent).astype(np.int32), (key % n_ent).astype(np.int32)
    cnt = rng.geometric(0.8, size=fs.shape[0]).astype(np.float64)     # co-occurrence count >= 1

    # passage -> entity edges (each passage names ~n_pe / n_pass entities)
    pe_p = rng.integers(0, n_pass, size=int(n_pe * (1.05 if topology == "uniform" else 1.15)) + 16, dtype=np.int64)
    pe_e = draw_entities(pe_p.shape[0])
    pkey = np.unique(pe_p * n_ent + pe_e)
    rng.shuffle(pkey)
    pkey = pkey[:n_pe]
    pe_p, pe_e = (pkey // n_ent).astype(np.int32), (pkey % n_ent).astype(np.int32)
    passage_vid = (n_ent + np.arange(n_pass)).astype(np.int32)

    # synonymy edges between entities
    sy_a = draw_entities(max(n_syn, 0))
    sy_b = draw_entities(max(n_syn, 0))
    ok = sy_a != sy_b
    sy_a, sy_b = sy_a[ok].astype(np.int32), sy_b[ok].astype(np.int32)
    sy_w = 0.8 + 0.2 * rng.random(sy_a.shape[0])

    edge_src = np.concatenate([fs, fo, passage_vid[pe_p], sy_a]).astype(np.int32)
    edge_dst = np.concatenate([fo, fs, pe_e, sy_b]).astype(np.int32)
    edge_w = np.concatenate([cnt, cnt, np.ones(pe_p.shape[0]), sy_w])

    ent_chunk_count = np.zeros(n_nodes, dtype=np.int32)
    np.add.at(ent_chunk_count, pe_e, 1)

    # for query planting: one passage adjacent to each fact's subject (or any passage)
    first_passage_of_ent = np.full(n_ent, -1, dtype=np.int32)
    first_passage_of_ent[pe_e[::-1]] = pe_p[::-1]
    fact_passage = first_passage_of_ent[fs]
    missing = fact_passage < 0
    fact_passage[missing] = rng.integers(0, n_pass, size=int(missing.sum()))

    return SynthKG(n_nodes, n_ent, n_pass, edge_src, edge_dst, edge_w, passage_vid, fs, fo,
                   ent_chunk_count, fact_passage.astype(np.int32))


def seeded_unit_vectors(seeds, dim: int) -> np.ndarray:
    """Row i = normalised standard-normal vector drawn from ``default_rng(seeds[i])`` (fp32): how the committed
    MuSiQue-1k fixture (tests/golden/musique1k.npz, BASELINE config #1) stores its mock embeddings."""
    out = np.empty((len(seeds), dim), dtype=np.float32)
    for i, s in enumerate(seeds):
        v = np.random.default_rng(int(s)).standard_normal(dim)
        out[i] = (v / np.linalg.norm(v)).astype(np.float32)
    return out


def unit_rows(n: int, dim: int, seed: int, chunk: int = 1 << 16) -> np.ndarray:
    """[n, dim] fp32 unit-norm Gaussian rows, generated in chunks (bounded host memory)."""
    out = np.empty((n, dim), dtype=np.float32)
    rng = np.random.default_rng(seed)
    for lo in range(0, n, chunk):
        hi = min(n, lo + chunk)
        x = rng.standard_normal((hi - lo, dim), dtype=np.float32)
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        out[lo:hi] = x
    return out


def make_queries(kg: SynthKG, fact_emb: np.ndarray, passage_emb: np.ndarray, n_queries: int,
                 seed: int = 1, noise: float = 0.5):
    """Query pairs per SURVEY.md 8(d): q_fact = normalise(E_f[j] + noise*g), q_pass =
    normalise(E_p[i] + noise*g') with passage i adjacent to fact j's subject."""
    rng = np.random.default_rng(seed)
    dim = fact_emb.shape[1]
    j = rng.integers(0, kg.n_facts, size=n_queries)
    i = kg.fact_passage[j]

    def perturb(base):
        g = rng.standard_normal((n_queries, dim), dtype=np.float32)
        g /= np.linalg.norm(g, axis=1, keepdims=True)
        q = base + noise * g
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        return np.ascontiguousarray(q, dtype=np.float32)

    return perturb(fact_emb[j]), perturb(passage_emb[i]), j.astype(np.int32)


CONFIGS = {
    # name: (n_nodes, n_edges, dim, n_queries, topology)
    "C2": (100_000, 1_000_000, 768, 1_000, "uniform"),
    "C3": (1_000_000, 10_000_000, 768, 10_000, "uniform"),
    "C5": (10_000_000, 100_000_000, 1024, 128, "powerlaw"),
}
