"""Generates ``tests/golden/accelerate_glue150.npz`` for ``tests/test_accelerate.py::
test_accelerate_glue_against_reference_object``: the reference's own ``HippoRAG`` object after ``index()`` of the first
150 MuSiQue passages (64-d md5-seeded mock embeddings, identity filter), reduced to the state the drop-in reads, and
what the reference's own methods returned on it in the same sequence the test replays:

  ref_*     ``HippoRAG.retrieve`` (unmodified) on the first 12 MuSiQue questions, top 20
  ircot_*   ``HippoRAG.retrieve_ircot`` (the reference's serial loop) on the first 6, 3 steps, top 10, over the
            single-query retrieve of ``accelerate(rag, engine=OracleEngine())``, with ``FakeQALLM``
  ref10_*   ``HippoRAG.retrieve`` with linking_top_k = 10 on the first 4, after one edge was added to the graph

Documents are stored as passage indices, graph seeds and thoughts as JSON.

Needs a checkout of the reference:   HIPPORAG_REFERENCE_ROOT=<path> PYTHONHASHSEED=0 python tests/golden/make_accelerate_golden.py
"""
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_harness as H  # noqa: E402

N_DOCS, DIM, N_Q = 150, 64, 12


def main():
    import hipporag_b200
    from tests.test_accelerate import FakeQALLM, OracleEngine
    rag = H.build_reference_rag(tempfile.mkdtemp(prefix="hrag_acc_"), N_DOCS, DIM)
    from hipporag.prompts.linking import get_query_instruction
    questions = H.musique_questions(N_Q)
    ref = rag.retrieve(questions, num_to_retrieve=20)
    content_to_pidx = {rag.chunk_embedding_store.get_row(k)["content"]: i for i, k in enumerate(rag.passage_node_keys)}
    assert len(content_to_pidx) == len(rag.passage_node_keys)

    def ids(docs):
        return [content_to_pidx[d] for d in docs]
    rows = rag.fact_embedding_store.get_rows(rag.fact_node_keys)
    fact_contents = [rows[k]["content"] for k in rag.fact_node_keys]
    passage_contents = [rag.chunk_embedding_store.get_row(k)["content"] for k in rag.passage_node_keys]
    ent_keys = sorted(rag.ent_node_to_chunk_ids)
    gc = rag.global_config
    out = dict(
        dim=np.int32(DIM), questions=np.array(questions, dtype=str),
        q_fact_instruction=np.array(get_query_instruction("query_to_fact")),
        q_passage_instruction=np.array(get_query_instruction("query_to_passage")),
        vertex_names=np.array(rag.graph.vs["name"], dtype=str),
        graph_edges=np.asarray(rag.graph.get_edgelist(), dtype=np.int32).reshape(-1, 2),
        graph_weights=np.asarray(rag.graph.es["weight"], dtype=np.float64),
        passage_node_keys=np.array(rag.passage_node_keys, dtype=str),
        fact_node_keys=np.array(rag.fact_node_keys, dtype=str), fact_contents=np.array(fact_contents, dtype=str),
        fact_seed=np.array([H.text_seed(t) for t in fact_contents], dtype=np.uint64),
        passage_seed=np.array([H.text_seed(t) for t in passage_contents], dtype=np.uint64),
        ent_chunk_keys=np.array(ent_keys, dtype=str),
        ent_chunk_counts=np.array([len(rag.ent_node_to_chunk_ids[k]) for k in ent_keys], dtype=np.int32),
        config=np.array(json.dumps({k: getattr(gc, k) for k in (
            "retrieval_top_k", "linking_top_k", "damping", "passage_node_weight", "dataset")})),
        ref_ids=np.array([ids(r.docs) for r in ref], dtype=np.int32),
        ref_scores=np.array([np.asarray(r.doc_scores, dtype=np.float64) for r in ref]),
        ref_seeds=np.array(json.dumps([[list(f) for f in r.graph_seeds] for r in ref])),
    )
    # self-check: the stored seeds / instructions regenerate the embeddings the reference used
    assert np.array_equal(H.seeded_unit_vectors(out["fact_seed"][:8], DIM), rag.fact_embeddings[:8])
    assert np.array_equal(H.seeded_unit_vectors(out["passage_seed"][:8], DIM), rag.passage_embeddings[:8])
    assert np.array_equal(H.MockEmbeddingModel(DIM).batch_encode(questions[:2], instruction=str(out["q_fact_instruction"])),
                          np.stack([rag.query_to_embedding["triple"][q] for q in questions[:2]]))
    msgs = rag.prompt_template_manager.render(name=f"ircot_{gc.dataset}", prompt_user="P\n\nQuestion: Q\nThought:")
    assert msgs[-1]["content"] == "P\n\nQuestion: Q\nThought:"      # FakeQALLM reads the last message only

    hipporag_b200.accelerate(rag, engine=OracleEngine())
    rag.ready_to_retrieve = False
    rag.qa_llm = FakeQALLM()
    want = type(rag).retrieve_ircot(rag, questions[:6], max_qa_steps=3, num_to_retrieve=10)
    out["ircot_ids"] = np.array(json.dumps([ids(w.docs) for w in want]))
    out["ircot_scores"] = np.array(json.dumps([np.asarray(w.doc_scores, dtype=np.float64).tolist() for w in want]))
    out["ircot_thoughts"] = np.array(json.dumps([list(w.thoughts) for w in want]))
    rag.graph.add_edges([(rag.graph.vs["name"][0], rag.graph.vs["name"][1])], attributes={"weight": [0.5]})
    rag.ready_to_retrieve = False
    rag.rerank_filter = lambda q, c, i, len_after_rerank=None: (i[:len_after_rerank], c[:len_after_rerank], {})
    gc.linking_top_k = 10
    ref10 = type(rag).retrieve(rag, questions[:4], num_to_retrieve=10)
    out["ref10_seeds"] = np.array(json.dumps([[list(f) for f in r.graph_seeds] for r in ref10]))
    path = os.path.join(ROOT, "tests", "golden", "accelerate_glue150.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
