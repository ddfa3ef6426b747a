#!/usr/bin/env python
"""Paired fp16 sweep against the single one: ms per 32-column sweep of the compact-rhs Chebyshev sweep.

    python tools/paired_sweep_bench.py [--workloads C3,C5] [--sweeps 400] [--rounds 5]

`single` is k_sweep_h on one [N, 32] state (hrag_bench_sweep method 3); `paired` is k_sweep_h2, which walks each row
once for two states interleaved in one [N, 2, 32] buffer (method 4); its time per paired sweep is halved.  The two
alternate round by round on one handle, device events around `--sweeps` sweeps each; one JSON line per round and
variant, then a summary line per workload with each variant's min / median / max and the card's name and power limit
read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from bench import WORKLOADS  # noqa: E402

VARIANTS = (("single", 3, 1), ("paired", 4, 2))


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C3,C5")
    ap.add_argument("--sweeps", type=int, default=400)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    from hipporag_b200 import Engine, synth
    info = card()
    for name in args.workloads.split(","):
        w = WORKLOADS[name]
        kg = synth.make_kg(w["n_nodes"], w["n_edges"], seed=0, topology=w["topology"])
        e = Engine(0)
        e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
        e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        times = {v: [] for v, _, _ in VARIANTS}
        for r in range(args.rounds):
            for v, method, cols in VARIANTS:
                ms = e.bench_sweep(32, args.sweeps, method) / cols
                times[v].append(ms)
                print(json.dumps({"workload": name, "round": r, "variant": v, "ms_per_32col_sweep": round(ms, 4)}),
                      flush=True)
        summary = {"workload": name, "nodes": kg.n_nodes, "sweeps_per_measure": args.sweeps, **info}
        for v, ts in times.items():
            summary[v] = {"min": round(min(ts), 4), "median": round(float(np.median(ts)), 4), "max": round(max(ts), 4)}
        summary["paired"]["speedup_median"] = round(summary["single"]["median"] / summary["paired"]["median"], 3)
        print(json.dumps(summary), flush=True)
        e.close()


if __name__ == "__main__":
    main()
