#!/usr/bin/env python
"""Stage A's fact GEMM (K2, k_sim_tc with the fused top-8 epilogue) alone, then the chunk-overlap scan of
retrieve_resident.

    python tools/stage_a_bench.py [--workload C3] [--reps 5] [--steps 2] [--scan=0,-1,40,48] [--exact] [--out FILE]

K2 alone: stage_a on the workload's queries (1,024-query chunks) on the whole GPU; `ms_per_chunk` is the library's
sim_fact span (bf16 split of the queries + the GEMM, CUDA events) divided by the chunks, the median of --reps calls.
With the stage-A screen (the default; --exact runs the split GEMM over all facts instead) the span holds the screen
and the rescore; `screen_parts` then gives each part's kernel time per chunk from one profiled stage_a call
(torch.profiler): the screen (query split and bound, hi.hi GEMM), the candidate selection and staging, the split
rescore, the final selection, and the gated exact fallback (0 unless a chunk fell back).
The scan: one retrieve_resident step (the bench.py step) per G, CUDA events around --steps steps after a warm-up step;
G = 0 is the rule in overlap_ctas, G = -1 runs the chunks one after the other without the overlap.  The G values
alternate within each of --rounds rounds.  One JSON line per measurement, then a summary with the card's name and
power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import bench  # noqa: E402


def card():
    import torch
    info = {"gpu": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit"], info["max_sm_clock"] = [x.strip() for x in q.split(",")]
    except (OSError, ValueError, subprocess.TimeoutExpired):
        info["power_limit"] = "unknown"
    return info


PARTS = (("screen", ("k_split_bf16", "k_query_err", "k_sim_tc<false, 4>")),
         ("select", ("k_screen_select", "k_screen_stage", "k_screen_gather")),
         ("rescore", ("k_sim_tc<true, 3>",)),
         ("finish", ("k_screen_finish",)),
         ("exact_fallback", ("k_sim_tc<true, 1>", "k_merge_minmax_topk")))


def screen_parts(e, qf, chunks):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e.stage_a(qf, bench.LINK_TOP_K)
        torch.cuda.synchronize()
    ms = {name: 0.0 for name, _ in PARTS}
    for ev in prof.key_averages():
        for name, keys in PARTS:
            if any(k in ev.key for k in keys):
                ms[name] += ev.device_time_total / 1e3
    return {name: round(v / chunks, 3) for name, v in ms.items()}


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        with open(out, "a") as f:
            f.write(line + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="C3")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=1)
    ap.add_argument("--scan", default="0,-1,40,48,56,66")
    ap.add_argument("--out", default="")
    ap.add_argument("--exact", action="store_true", help="run stage A without the screen")
    args = ap.parse_args()
    import torch
    from hipporag_b200 import Engine
    device = torch.device("cuda", 0)
    info = card()
    w = bench.WORKLOADS[args.workload]
    Q = w["queries"]
    wl = bench.build_workload(args.workload, Q, device, 0)
    kg = wl.kg
    e = Engine(0)
    e.load_graph_csr(kg.n_nodes, *wl.csr)
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    e.load_embeddings(wl.fe, wl.pe)
    if args.exact:
        e.debug_exact_stage_a(True)
    chunks = -(-Q // 1024)
    summary = {"workload": args.workload, "queries": Q, "facts": kg.n_facts, "dim": w["dim"], **info}

    # ---- K2 alone
    qf = wl.qf.cpu().numpy()
    e.stage_a(qf, bench.LINK_TOP_K)                     # warm-up
    k2 = []
    for r in range(args.reps):
        e.reset_stats()
        e.stage_a(qf, bench.LINK_TOP_K)
        ms = e.stats()["ms_sim_fact"] / chunks
        k2.append(ms)
        emit({"what": "k2_alone", "rep": r, "ms_per_chunk": round(ms, 3)}, args.out)
    flop = 2.0 * 4 * 1024 * kg.n_facts * w["dim"]      # four split products per 1,024-query chunk
    med = float(np.median(k2))
    summary["k2_alone_ms_per_chunk"] = {"min": round(min(k2), 3), "median": round(med, 3), "max": round(max(k2), 3)}
    summary["k2_alone_tflops_issued"] = round(flop / (med * 1e-3) / 1e12, 1)
    summary["stage_a_fallbacks"] = e.stats()["stage_a_fallbacks"]
    if not args.exact:
        summary["screen_parts_ms_per_chunk"] = screen_parts(e, qf, chunks)

    # ---- G scan of retrieve_resident
    out_ids = torch.empty((Q, bench.TOPK), dtype=torch.int32, device=device)
    out_scores = torch.empty((Q, bench.TOPK), dtype=torch.float32, device=device)
    stream = torch.cuda.ExternalStream(e.stream_ptr, device=device)
    gs = [int(g) for g in args.scan.split(",") if g.strip()]
    steps = {g: [] for g in gs}
    for rnd in range(args.rounds):
        for g in gs:
            e.debug_sim_ctas(g)

            def step():
                e.retrieve_resident(wl.qf, wl.qp, out_ids, out_scores, bench.DAMPING, bench.PNW, bench.LINK_TOP_K,
                                    bench.TOPK)
            step()
            torch.cuda.synchronize()
            e.reset_stats()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(args.steps):
                step()
            e1.record(stream)
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.steps
            st = e.stats()
            sweeps = max(st["ppr_sweeps"], 1)
            rec = {"what": "scan", "round": rnd, "G": g, "ms_per_step": round(ms, 1), "qps": round(Q / ms * 1e3, 1),
                   "ms_sim_fact": round(st["ms_sim_fact"] / args.steps, 1), "ms_ppr": round(st["ms_ppr"] / args.steps, 1),
                   "ms_ppr_per_sweep": round(st["ms_ppr"] / sweeps, 4)}
            steps[g].append(ms)
            emit(rec, args.out)
    if gs:
        e.debug_sim_ctas(0)
    summary["scan_ms_per_step"] = {str(g): {"min": round(min(v), 1), "max": round(max(v), 1)} for g, v in steps.items()}
    emit(summary, args.out)
    e.close()


if __name__ == "__main__":
    main()
