#!/usr/bin/env python
"""Cost of retrieve() at PRPACK accuracy: Engine.stage_b (fp32 / mixed PPR, tol 1e-6) against Engine.stage_b_f64
(float64 reset, PPR by iterative refinement to 1e-10, float64 gather and top-k), per call, on the C1 graph
(MuSiQue-1k, its 64 queries) and the C3 graph (1M nodes / 10M edges) at B in {16, 256, 1024}.

    python tools/stage_b_f64_bench.py [--workloads C1,C3] [--runs 3]

Stage A runs once per (workload, B); its kept facts feed both stage B variants.  One JSON line per (workload, B,
variant): best-of-runs ms per call (host clock around the call, which ends in a device synchronise), the library's
device-timed ms_seed / ms_ppr / ms_topk of that run, the sweeps per call (fp64: refinement rounds per sub-batch), the
error bound, and the card name and power limit read in the same run.
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from tools.ppr_f64_bench import card  # noqa: E402


def setup(name):
    """(engine, q_fact pool, q_pass pool, damping, pnw, linking_top_k)"""
    from hipporag_b200 import Engine, synth
    from bench import WORKLOADS
    e = Engine(0)
    if name == "C1":
        from oracle.ref_harness import seeded_unit_vectors
        g = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                                 "musique1k.npz"))
        dim = int(g["dim"])
        e.load_graph(int(g["n_nodes"]), g["edge_src"], g["edge_dst"], g["edge_w"])
        e.load_tables(g["passage_vid"], g["fact_subj_vid"], g["fact_obj_vid"], g["ent_chunk_count"])
        e.load_embeddings(seeded_unit_vectors(g["fact_seed"], dim), seeded_unit_vectors(g["passage_seed"], dim))
        return (e, seeded_unit_vectors(g["qfact_seed"], dim), seeded_unit_vectors(g["qpass_seed"], dim),
                float(g["damping"]), float(g["passage_node_weight"]), int(g["linking_top_k"]))
    w = WORKLOADS[name]
    kg = synth.make_kg(w["n_nodes"], w["n_edges"], seed=0, topology=w["topology"])
    fe, pe = synth.unit_rows(kg.n_facts, w["dim"], 1), synth.unit_rows(kg.n_pass, w["dim"], 2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 1024, seed=3)
    e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    e.load_embeddings(fe, pe)
    return e, qf, qp, 0.5, 0.05, 5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C1,C3")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--topk", type=int, default=200)
    args = ap.parse_args()
    gpu, limits = card()
    for wl in args.workloads.split(","):
        e, qf, qp, a, pnw, ltk = setup(wl)
        for B in ((64,) if wl == "C1" else (16, 256, 1024)):
            idx, score, _ = e.stage_a(qf[:B], ltk)
            for variant in ("stage_b", "stage_b_f64"):
                fn = getattr(e, variant)
                fn(qp[:B], idx, score, None, a, pnw, ltk, args.topk)          # warm-up: allocations, module load
                best = None
                for _ in range(args.runs):
                    e.reset_stats()
                    t = time.perf_counter()
                    fn(qp[:B], idx, score, None, a, pnw, ltk, args.topk)
                    ms = (time.perf_counter() - t) * 1e3
                    if best is None or ms < best[0]:
                        best = (ms, e.stats())
                ms, st = best
                n_sub = -(-B // 16)
                print(json.dumps({
                    "workload": wl, "B": B, "variant": variant, "ms_per_call": round(ms, 3),
                    "ms_per_query": round(ms / B, 4), "ms_sim_passage": round(st["ms_sim_passage"], 3),
                    "ms_seed": round(st["ms_seed"], 3), "ms_ppr": round(st["ms_ppr"], 3),
                    "ms_topk": round(st["ms_topk"], 3), "sweeps": st["ppr_sweeps"],
                    # fp64: a round is one fp32 solve + one residual sweep; the residual sweeps are 1 in (iters + 1)
                    "rounds_per_sub_batch": None if variant == "stage_b" else
                    round(st["ppr_sweeps"] / n_sub / (1 + _fp32_sweeps(a)), 2),
                    "error_bound": st["ppr_error_bound"], "gpu": gpu, "power_limit,max_sm_clock": limits}),
                    flush=True)
        e.close()


def _fp32_sweeps(damping):
    from hipporag_b200.engine import plan_sweeps
    return plan_sweeps(damping, 1e-6, 0, 16)["fp32_sweeps"]


if __name__ == "__main__":
    main()
