"""Generates ``tests/golden/dropin_tables120.npz``: the state of the reference's own ``HippoRAG`` object that
``hipporag_b200.accelerate.extract_tables`` reads (graph, node names, passage vertices, fact rows, entity -> chunk
counts) after ``index()`` of the first 120 MuSiQue passages, and the integer tables ``oracle.ref_harness.extract_tables``
derives from that object -- so the drop-in's extraction is checked against the reference's run without the reference.

Needs a checkout of the reference:   HIPPORAG_REFERENCE_ROOT=<path> PYTHONHASHSEED=0 python tests/golden/make_dropin_golden.py
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle import ref_harness as H  # noqa: E402

N_DOCS, DIM = 120, 32


def main():
    rag = H.build_reference_rag(tempfile.mkdtemp(prefix="hrag_tb_"), N_DOCS, DIM)
    want = H.extract_tables(rag)                    # prepares the retrieval objects
    edges = np.asarray(rag.graph.get_edgelist(), dtype=np.int32).reshape(-1, 2)
    rows = rag.fact_embedding_store.get_rows(rag.fact_node_keys)
    ent_keys = sorted(rag.ent_node_to_chunk_ids)
    out = dict(
        vertex_names=np.array(rag.graph.vs["name"], dtype=str),
        graph_edges=edges, graph_weights=np.asarray(rag.graph.es["weight"], dtype=np.float64),
        passage_node_idxs=np.asarray(rag.passage_node_idxs, dtype=np.int32),
        fact_node_keys=np.array(rag.fact_node_keys, dtype=str),
        fact_contents=np.array([rows[k]["content"] for k in rag.fact_node_keys], dtype=str),
        ent_chunk_keys=np.array(ent_keys, dtype=str),
        ent_chunk_counts=np.array([len(rag.ent_node_to_chunk_ids[k]) for k in ent_keys], dtype=np.int32),
        want_n_nodes=np.int64(want["n_nodes"]),
        want_fact_texts=np.array(want["fact_texts"], dtype=str),
        **{"want_" + k: np.asarray(want[k]) for k in ("edge_src", "edge_dst", "edge_w", "passage_vid",
                                                       "fact_subj_vid", "fact_obj_vid", "ent_chunk_count")},
    )
    path = os.path.join(ROOT, "tests", "golden", "dropin_tables120.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
