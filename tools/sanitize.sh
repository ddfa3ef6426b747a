#!/bin/bash
# compute-sanitizer passes over a small end-to-end run of every kernel family (SURVEY.md 5: race detection).
# Usage (on an H100): bash tools/sanitize.sh [memcheck|racecheck|synccheck|initcheck]
set -u
TOOL=${1:-memcheck}
cat > /tmp/hrag_sanitize_driver.py <<'PY'
import numpy as np, sys, os
sys.path.insert(0, os.getcwd())
import hipporag_b200 as hb
from hipporag_b200 import synth
kg = synth.make_kg(3000, 30000, seed=5)
d = 64
fe, pe = synth.unit_rows(kg.n_facts, d, 1), synth.unit_rows(kg.n_pass, d, 2)
qf, qp, _ = synth.make_queries(kg, fe, pe, 40, seed=3)
# a hub row > 256 nnz so the long-row kernels run too
src = np.concatenate([kg.edge_src, np.zeros(400, np.int32)]); dst = np.concatenate([kg.edge_dst, np.arange(1, 401, dtype=np.int32)])
w = np.concatenate([kg.edge_w, np.ones(400)])
r = hb.B200Retriever(kg.n_nodes, src, dst, w, kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count, fe, pe)
for prec in (hb.PPR_MIXED, hb.PPR_FP32):
    for sim in (hb.SIM_BF16X3, hb.SIM_BF16, hb.SIM_FP32):
        r.engine.set_options(ppr_precision=prec, sim_mode=sim)
        ids, sc, _, _ = r.retrieve(qf, qp, topk=50)
        ids2, sc2, _, _ = r.retrieve(qf[:5], qp[:5], topk=50)
r.engine.set_options(ppr_precision=hb.PPR_MIXED, sim_mode=hb.SIM_BF16X3)
R = np.random.default_rng(0).random((3, kg.n_nodes), dtype=np.float32)
r.engine.ppr(R)
r.engine.ppr(np.random.default_rng(1).random((20, kg.n_nodes), dtype=np.float32), damping=0.85)
r.engine.similarity(1, qp[:3])
# round-2 kernels: linking_top_k > 8 (radix select path + 64 seed slots), threshold KNN epilogue
idx, score, nv = r.engine.stage_a(qf, 10)
r.engine.stage_b(qp, idx, score, link_top_k=10, topk=50)
r.engine.knn_threshold(0, fe[:200], 0.3, 64)
# in-place index updates (index_update.cu): an append and a delete on a mutable handle, then one mixed stage B
m = hb.B200Retriever(kg.n_nodes, src, dst, w, kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count,
                     fe, pe, engine=hb.Engine(0, mutable=True)).engine
N = kg.n_nodes
m.append(3, np.array([N, N + 1, 5], np.int32), np.array([7, 9, N + 2], np.int32), np.array([1.0, 0.5, 2.0]),
         np.array([N + 2], np.int32), np.array([N, 3], np.int32), np.array([N + 1, -1], np.int32),
         np.r_[kg.ent_chunk_count, [1, 2, 0]].astype(np.int32), fe[:2], pe[:1])
m.delete(np.array([0, 11, N + 1], np.int32), np.array([1, 4], np.int32),
         np.delete(np.r_[kg.ent_chunk_count, [1, 2, 0]], [0, 11, N + 1]).astype(np.int32))
idx, score, nv = m.stage_a(qf, 5)
m.stage_b(qp, idx, score, topk=50)
# the resident synonymy KNN (knn_index.cu): a build with overflowing rows, then an append + delete update
rng = np.random.default_rng(4)
ent = rng.choice([-1.0, 1.0], size=(1500, 64)).astype(np.float32)
ent[:600, :48] = ent[0, :48]
ent /= 8
m.knn_index_update(ent, None, 0.375, 128)
m.knn_index_update(np.concatenate([ent[3:], ent[:40]]), np.arange(3, 1500), 0.375, 128)
m.knn_index_read()
# fact planes in pinned host memory (fact_stream.cu): a 256-row-slice ring, fused and materialised stage A, similarity
f = hb.B200Retriever(kg.n_nodes, src, dst, w, kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count,
                     fe, pe, engine=hb.Engine(0, fact_device_bytes=2 * 256 * d * 4)).engine
f.stage_a(qf, 5)
f.stage_a(qf, 10)
f.similarity(0, qf[:3])
f.topk_similarity(0, qf[:3], 40)
# the hi fact plane resident and the lo plane in mapped pinned host memory (HRAG_FACT_LO_ON_HOST): the screen with its
# lo gather over PCIe (k = 5), a chunk that falls back (copies of row 1024 in 12 tiles saturate more tiles than a query
# may list) and reruns with the lo plane streamed, the streamed k = 10 path and similarity(0)
F2 = 65_536 + 37
rng = np.random.default_rng(6)
fe2 = rng.standard_normal((F2, d)).astype(np.float32)
fe2 /= np.linalg.norm(fe2, axis=1, keepdims=True)
for t in range(4, 16):
    fe2[t * 256:t * 256 + 10] = fe2[1024]
q2 = fe2[rng.integers(4096, F2, 40)] + 0.05 * rng.standard_normal((40, d)).astype(np.float32)
s = hb.Engine(0, fact_device_bytes=F2 * d * 2 + 2 * 256 * d * 2, fact_lo_on_host=True)
s.load_embeddings(fe2, pe)
assert s.fact_planes_info()["on_host"] == 2
s.stage_a(q2, 5)
q2[7] = fe2[1024]
s.reset_stats()
s.stage_a(q2, 5)
assert s.stats()["stage_a_fallbacks"] == 1
s.stage_a(q2, 10)
s.similarity(0, q2[:3])
# the screen with the lo plane on the host at each cap's last slot (tests/test_gpu_screen_caps.py): 256 candidates
# for every query of an m-tile, 8 saturated tiles (the ragged last one among them), 48 staged rows in one column and
# in every column of an m-tile; each exact, without a fallback
from tests import test_gpu_screen_caps as caps
for name in ("candidates at cap", "saturated tiles at cap", "48 staged rows in a column",
             "48 saturated tiles in an m-tile"):
    w = caps.CASES[name][0]()
    c = hb.Engine(0, fact_device_bytes=caps._lo_budget(), fact_lo_on_host=True)
    c.load_embeddings(w["E"], w["E"][:4])
    c.reset_stats()
    idx, _, _ = c.stage_a(w["Q"][w["calls"][name]], 8)
    assert c.stats()["stage_a_fallbacks"] == 0, name
    assert np.array_equal(idx, caps.exact_outputs(caps.CASES[name][0])[0][w["calls"][name]]), name
    c.close()
print("driver ok", ids.shape)
PY
compute-sanitizer --tool $TOOL --error-exitcode 7 python /tmp/hrag_sanitize_driver.py 2>&1 | tail -15
echo "sanitizer($TOOL) exit: $?"
