#!/usr/bin/env python
"""The first sweep of a paired stage-B solve in both forms: ms per paired sweep (two 32-column sub-batches).

    python tools/first_sweep_bench.py [--workloads C3,C5] [--sweeps 400] [--rounds 5]

`dense` gathers the dense first iterate x0 from the [N, 2, 32] pair buffer (hrag_bench_sweep method 5, the form
node-range sharding and Engine.debug_dense_first_sweep keep); `compact` reads the compact right-hand side through the
slot maps of the passages and loads nothing for the other columns (method 6, stage B's default on one GPU).  Both are
the plain (non-Chebyshev) sweep of k_sweep_h2.  The two alternate round by round on one handle, device events around
`--sweeps` sweeps each; one JSON line per round and variant, then a summary line per workload with each variant's
min / median / max and the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from bench import WORKLOADS  # noqa: E402
from tools.paired_sweep_bench import card  # noqa: E402

VARIANTS = (("dense", 5), ("compact", 6))


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
        times = {v: [] for v, _ in VARIANTS}
        for r in range(args.rounds):
            for v, method in VARIANTS:
                ms = e.bench_sweep(32, args.sweeps, method)
                times[v].append(ms)
                print(json.dumps({"workload": name, "round": r, "variant": v, "ms_per_paired_sweep": round(ms, 4)}),
                      flush=True)
        summary = {"workload": name, "nodes": kg.n_nodes, "sweeps_per_measure": args.sweeps, **info}
        for v, ts in times.items():
            summary[v] = {"min": round(min(ts), 4), "median": round(float(np.median(ts)), 4), "max": round(max(ts), 4)}
        summary["compact"]["speedup_median"] = round(summary["dense"]["median"] / summary["compact"]["median"], 3)
        print(json.dumps(summary), flush=True)
        e.close()


if __name__ == "__main__":
    main()
