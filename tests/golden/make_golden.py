"""Generates ``tests/golden/musique1k.npz`` by running the reference's own unmodified
``HippoRAG.index()`` / ``retrieve()`` (via ``oracle/ref_harness.py``) on BASELINE config #1:
the first 1,000 MuSiQue passages of the shipped OpenIE file, the first 64 MuSiQue questions,
768-d md5-seeded mock embeddings, identity recognition-memory filter.

Needs a checkout of the reference:   HIPPORAG_REFERENCE_ROOT=<path> PYTHONHASHSEED=0 python tests/golden/make_golden.py

What the file pins: rows A-D and F of SURVEY.md 8(a) come from the reference's code
verbatim.  Row E (PPR) went through ``oracle/fake_igraph.py`` -- python-igraph is not
installable offline -- so the PPR scores in it are the oracle's float64 direct solve, NOT
PRPACK's ("parity unpinned" at that boundary).

Embeddings are not stored (33 MB); the fixture keeps their 64-bit seeds and tests rebuild
them with ``oracle.ref_harness.seeded_unit_vectors``.
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_harness as H  # noqa: E402

N_DOCS, N_Q, DIM, TOPK = 1000, 64, 768, 200


def main():
    H.install_stubs()
    from hipporag.prompts.linking import get_query_instruction
    tmp = tempfile.mkdtemp(prefix="hrag_golden_")
    rag = H.build_reference_rag(tmp, N_DOCS, DIM)
    questions = H.musique_questions(N_Q)
    tables = H.extract_tables(rag)

    captured = {"reset": [], "facts_idx": [], "fact_scores": []}
    orig_run_ppr = rag.run_ppr
    orig_rerank = rag.rerank_facts

    def run_ppr_spy(reset_prob, damping=0.5):
        captured["reset"].append(np.array(reset_prob, dtype=np.float64))
        return orig_run_ppr(reset_prob, damping)

    def rerank_spy(query, query_fact_scores):
        idx, facts, log = orig_rerank(query, query_fact_scores)
        captured["facts_idx"].append(np.array(idx, dtype=np.int32))
        captured["fact_scores"].append(np.array([query_fact_scores[i] for i in idx], dtype=np.float32))
        return idx, facts, log

    rag.run_ppr = run_ppr_spy
    rag.rerank_facts = rerank_spy
    sols = rag.retrieve(questions, num_to_retrieve=TOPK)

    key_to_pidx = {rag.chunk_embedding_store.get_row(k)["content"]: i for i, k in enumerate(rag.passage_node_keys)}
    top_ids = np.array([[key_to_pidx[d] for d in s.docs] for s in sols], dtype=np.int32)
    top_scores = np.array([np.asarray(s.doc_scores, dtype=np.float64) for s in sols])
    reset = np.stack(captured["reset"])                       # [Q, N] float64
    ent_mask = np.ones(tables["n_nodes"], dtype=bool)
    ent_mask[tables["passage_vid"]] = False
    seed_vid = np.full((N_Q, 8), -1, dtype=np.int32)
    seed_w = np.zeros((N_Q, 8), dtype=np.float64)
    for q in range(N_Q):
        nz = np.nonzero(reset[q] * ent_mask)[0]
        seed_vid[q, :len(nz)] = nz
        seed_w[q, :len(nz)] = reset[q, nz]
    passage_reset = reset[:, tables["passage_vid"]]           # [Q, P] = 0.05 * minmax(dpr)

    q_fact_instr = get_query_instruction("query_to_fact")
    q_pass_instr = get_query_instruction("query_to_passage")
    out = dict(
        n_nodes=np.int64(tables["n_nodes"]), dim=np.int32(DIM), topk=np.int32(TOPK),
        edge_src=tables["edge_src"], edge_dst=tables["edge_dst"], edge_w=tables["edge_w"],
        passage_vid=tables["passage_vid"], fact_subj_vid=tables["fact_subj_vid"],
        fact_obj_vid=tables["fact_obj_vid"], ent_chunk_count=tables["ent_chunk_count"],
        fact_seed=np.array([H.text_seed(t) for t in tables["fact_texts"]], dtype=np.uint64),
        passage_seed=np.array([H.text_seed(t) for t in tables["passage_texts"]], dtype=np.uint64),
        qfact_seed=np.array([H.text_seed(t, q_fact_instr) for t in questions], dtype=np.uint64),
        qpass_seed=np.array([H.text_seed(t, q_pass_instr) for t in questions], dtype=np.uint64),
        ref_fact_idx=np.stack(captured["facts_idx"]), ref_fact_score=np.stack(captured["fact_scores"]),
        ref_seed_vid=seed_vid, ref_seed_w=seed_w,
        ref_passage_reset=passage_reset.astype(np.float32),
        ref_top_ids=top_ids, ref_top_scores=top_scores,
        damping=np.float64(rag.global_config.damping),
        passage_node_weight=np.float64(rag.global_config.passage_node_weight),
        linking_top_k=np.int32(rag.global_config.linking_top_k),
    )
    # self-check: the stored seeds regenerate the embeddings the reference used
    assert np.array_equal(H.seeded_unit_vectors(out["fact_seed"][:16], DIM), rag.fact_embeddings[:16])
    assert np.array_equal(H.seeded_unit_vectors(out["passage_seed"][:16], DIM), rag.passage_embeddings[:16])
    assert np.array_equal(H.seeded_unit_vectors(out["qfact_seed"][:4], DIM),
                          np.stack([rag.query_to_embedding["triple"][q] for q in questions[:4]]))
    path = os.path.join(ROOT, "tests", "golden", "musique1k.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes;",
          "N=%d E=%d F=%d P=%d" % (tables["n_nodes"], len(tables["edge_w"]), len(tables["fact_texts"]),
                                   len(tables["passage_texts"])))


if __name__ == "__main__":
    main()
