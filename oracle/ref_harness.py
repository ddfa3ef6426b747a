"""Runs the reference's own, unmodified ``HippoRAG`` class offline.
TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``); usable only where a checkout of the
reference exists, named by the ``HIPPORAG_REFERENCE_ROOT`` environment variable.  The tests never
need it: what they compare with the reference's run is stored under ``tests/golden/``.

Recipe (SURVEY.md appendix B): inert stub modules for the network/LLM dependencies
that are not installed, ``oracle/fake_igraph.py`` registered as ``igraph``, the shipped
OpenIE results copied where ``HippoRAG.py:178`` looks for them so ``index()`` makes no
LLM call (``:295-300``), an md5-seeded mock embedder (pattern of
``tests/integration/run_vector_stores.py:34-44``, made process-independent) injected via
``embedding_model=`` (``HippoRAG.py:148-153``) and an identity recognition-memory filter
(``rerank.py:108-112`` signature).
"""
from __future__ import annotations

import hashlib
import json
import os
import sys
import types

import numpy as np

REFERENCE_ROOT = os.environ.get("HIPPORAG_REFERENCE_ROOT", "")


class _Anything:
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Anything()

    def __getattr__(self, name):
        return _Anything()


class _StubModule(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return type(name, (_Anything,), {})


def install_stubs():
    for name in ["litellm", "boto3", "botocore", "botocore.auth", "botocore.awsrequest",
                 "botocore.exceptions", "gritlm", "sentence_transformers"]:
        if name not in sys.modules:
            m = _StubModule(name)
            m.__path__ = []
            sys.modules[name] = m
    from . import fake_igraph
    try:
        import igraph  # noqa: F401  (a real igraph wins when it exists)
    except Exception:
        fake_igraph.install()
    src = os.path.join(REFERENCE_ROOT, "src")
    if src not in sys.path:
        sys.path.insert(0, src)


def text_seed(text: str, instruction: str = "") -> int:
    """64-bit seed of a text (+ instruction), process-independent."""
    h = hashlib.md5((instruction + "|" + text).encode("utf-8")).digest()
    return int.from_bytes(h[:8], "little")


def seeded_unit_vectors(seeds, dim: int) -> np.ndarray:
    """Row i = normalised standard-normal vector drawn from ``default_rng(seeds[i])`` (fp32).
    The golden fixture stores only the seeds; tests regenerate the vectors with this."""
    out = np.empty((len(seeds), dim), dtype=np.float32)
    for i, s in enumerate(seeds):
        v = np.random.default_rng(int(s)).standard_normal(dim)
        out[i] = (v / np.linalg.norm(v)).astype(np.float32)
    return out


class MockEmbeddingModel:
    """``batch_encode(texts, instruction=..., norm=...)`` -> [n, dim] fp32 unit vectors."""

    def __init__(self, dim: int = 768):
        self.dim = dim
        self.embedding_dim = dim

    def batch_encode(self, texts, instruction: str = "", norm: bool = True, **kwargs):
        if isinstance(texts, str):
            texts = [texts]
        return seeded_unit_vectors([text_seed(t, instruction or "") for t in texts], self.dim)


class StubLLM:
    def __init__(self, *a, **k):
        self.llm_name = "stub"

    def infer(self, *a, **k):
        raise RuntimeError("the offline harness must never call an LLM")

    batch_infer = infer


def identity_filter(query, candidate_items, candidate_indices, len_after_rerank=None):
    return candidate_indices[:len_after_rerank], candidate_items[:len_after_rerank], {}


def build_reference_rag(save_dir: str, n_docs: int, dim: int = 768,
                        openie_file: str = "openie_results_ner_gpt-4o-mini.json"):
    """index() the first ``n_docs`` MuSiQue passages with the reference's own code."""
    install_stubs()
    from hipporag import HippoRAG                      # the reference package
    from hipporag.utils.config_utils import BaseConfig

    with open(os.path.join(REFERENCE_ROOT, "outputs", "musique", openie_file)) as f:
        openie = json.load(f)
    openie["docs"] = openie["docs"][:n_docs]
    os.makedirs(save_dir, exist_ok=True)
    with open(os.path.join(save_dir, "openie_results_ner_gpt-4o-mini.json"), "w") as f:
        json.dump(openie, f)
    docs = [d["passage"] for d in openie["docs"]]

    cfg = BaseConfig(save_dir=save_dir, llm_name="gpt-4o-mini", embedding_model_name="mock",
                     dataset="musique")
    rag = HippoRAG(global_config=cfg, extraction_llm=StubLLM(), embedding_model=MockEmbeddingModel(dim))
    rag.rerank_filter = identity_filter
    rag.index(docs)
    return rag


def musique_questions(n: int):
    with open(os.path.join(REFERENCE_ROOT, "reproduce", "dataset", "musique.json")) as f:
        return [s["question"] for s in json.load(f)[:n]]


def extract_tables(rag):
    """Integer tables equivalent to the dicts ``prepare_retrieval_objects`` built
    (``HippoRAG.py:1287-1389``) -- what the engine uploads."""
    from hipporag.utils.misc_utils import compute_mdhash_id
    if not rag.ready_to_retrieve:
        rag.prepare_retrieval_objects()
    n = rag.graph.vcount()
    name_to_vid = rag.node_name_to_vertex_idx
    edges = np.asarray(rag.graph.get_edgelist(), dtype=np.int32).reshape(-1, 2)
    weights = np.asarray(rag.graph.es["weight"], dtype=np.float64)
    passage_vid = np.asarray(rag.passage_node_idxs, dtype=np.int32)
    fact_rows = rag.fact_embedding_store.get_rows(rag.fact_node_keys)
    F = len(rag.fact_node_keys)
    subj = np.full(F, -1, dtype=np.int32)
    obj = np.full(F, -1, dtype=np.int32)
    fact_texts = []
    for i, key in enumerate(rag.fact_node_keys):
        content = fact_rows[key]["content"]
        fact_texts.append(content)
        f = eval(content)                                    # HippoRAG.py:1693
        subj[i] = name_to_vid.get(compute_mdhash_id(f[0].lower(), prefix="entity-"), -1)  # :1584,:1591-1595
        obj[i] = name_to_vid.get(compute_mdhash_id(f[2].lower(), prefix="entity-"), -1)
    cnt = np.zeros(n, dtype=np.int32)
    for key, chunks in rag.ent_node_to_chunk_ids.items():   # :1598-1601
        vid = name_to_vid.get(key)
        if vid is not None:
            cnt[vid] = len(chunks)
    passage_texts = [rag.chunk_embedding_store.get_row(k)["content"] for k in rag.passage_node_keys]
    return dict(n_nodes=n, edge_src=edges[:, 0].copy(), edge_dst=edges[:, 1].copy(), edge_w=weights,
                passage_vid=passage_vid, fact_subj_vid=subj, fact_obj_vid=obj, ent_chunk_count=cnt,
                fact_texts=fact_texts, passage_texts=passage_texts)
