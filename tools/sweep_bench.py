#!/usr/bin/env python
"""K1 micro-benchmark: ms per SpMM sweep and achieved algorithmic GB/s per batch width.
    python tools/sweep_bench.py [C2|C3] [--sweeps 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from bench import WORKLOADS, measured_peaks, ppr_bytes_per_sweep  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("workload", nargs="?", default="C3")
    ap.add_argument("--sweeps", type=int, default=20)
    ap.add_argument("--widths", default="4,8,16,32,64")
    ap.add_argument("--topology", default="")
    ap.add_argument("--mixed", action="store_true")
    ap.add_argument("--nodes", type=int, default=0)
    ap.add_argument("--edges", type=int, default=0)
    args = ap.parse_args()
    from hipporag_b200 import Engine, PPR_CHEBYSHEV, PPR_POWER, synth
    from hipporag_b200.engine import build_transition_csr
    w = WORKLOADS.get(args.workload) or dict(n_nodes=10_000_000, n_edges=100_000_000, topology="powerlaw")
    if args.nodes:
        w = dict(w, n_nodes=args.nodes, n_edges=args.edges or 10 * args.nodes)
    kg = synth.make_kg(w["n_nodes"], w["n_edges"], seed=0, topology=args.topology or w["topology"])
    row_ptr, col, val = build_transition_csr(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    deg = np.diff(row_ptr)
    print(f"# {args.workload}: N={kg.n_nodes} nnz={col.shape[0]} deg mean {deg.mean():.1f} max {deg.max()}", flush=True)
    e = Engine(0)
    e.load_graph_csr(kg.n_nodes, row_ptr, col, val)
    peak, src = measured_peaks()
    if args.mixed:
        # the fp16 Chebyshev sweep with a dense [N, 32] rhs (hrag_ppr) and with the compact rhs of stage B
        e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
        by = ppr_bytes_per_sweep(kg.n_nodes, col.shape[0], 32) + kg.n_nodes * 32 * 4
        for name, m in (("mixed-fp16 chebyshev sweep, dense rhs", 2), ("mixed-fp16 chebyshev sweep, compact rhs", 3)):
            ms = e.bench_sweep(32, args.sweeps, m)
            print(json.dumps({"workload": args.workload, "B": 32, "method": name,
                              "ms_per_sweep": round(ms, 4), "alg_GBps": round(by / (ms * 1e-3) / 1e9, 1),
                              "frac_of_peak": round(by / (ms * 1e-3) / 1e9 / peak, 3),
                              "us_per_query_sweep": round(1000 * ms / 32, 2)}), flush=True)
    for B in [int(x) for x in args.widths.split(",") if x]:
        for name, m in (("power", PPR_POWER), ("chebyshev", PPR_CHEBYSHEV)):
            ms = e.bench_sweep(B, args.sweeps, m)
            by = ppr_bytes_per_sweep(kg.n_nodes, col.shape[0], B) + (kg.n_nodes * B * 4 if m == PPR_CHEBYSHEV else 0)
            gbs = by / (ms * 1e-3) / 1e9
            print(json.dumps({"workload": args.workload, "B": B, "method": name, "ms_per_sweep": round(ms, 4),
                              "alg_GBps": round(gbs, 1), "frac_of_peak": round(gbs / peak, 3),
                              "us_per_query_sweep": round(1000 * ms / B, 2),
                              "ps_per_nnz_col": round(1e9 * ms / B / col.shape[0], 3)}), flush=True)


if __name__ == "__main__":
    main()
