#!/usr/bin/env python
"""Cost of run_ppr at PRPACK accuracy: hrag_ppr (fp32) against hrag_ppr_f64 (float64 by iterative refinement), per call
and per stage, on the C1 graph (MuSiQue-1k) and the C3 graph (1M nodes / 10M edges), B in {1, 16}.

    python tools/ppr_f64_bench.py [--workloads C1,C3] [--reps 10]

One JSON line per (workload, B, solver): wall ms per call (host clock around the call, which ends in a device
synchronise), ms_solve (the library's device-timed PPR stage), ms_h2d / ms_d2h (a pageable host <-> device copy of the
same byte count, timed separately), the rounds and error bound of the fp64 solve, and the card name and power limit
read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from bench import WORKLOADS  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:          # the number still stands, but without its power limit
        q = f"unknown ({e})"
    return name, q


def copy_ms(nbytes, reps):
    """Pageable host -> device and device -> host copy of nbytes (what the ppr calls move), ms each."""
    import torch
    h = np.ones(nbytes // 8, np.float64)
    d = torch.from_numpy(h).cuda()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        d.copy_(torch.from_numpy(h))
    torch.cuda.synchronize()
    h2d = (time.perf_counter() - t) * 1e3 / reps
    t = time.perf_counter()
    for _ in range(reps):
        d.cpu()
    torch.cuda.synchronize()
    return h2d, (time.perf_counter() - t) * 1e3 / reps


def graph(name):
    from hipporag_b200 import synth
    if name == "C1":
        g = np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                                 "musique1k.npz"))
        return int(g["n_nodes"]), g["edge_src"], g["edge_dst"], g["edge_w"], g["passage_vid"]
    w = WORKLOADS[name]
    kg = synth.make_kg(w["n_nodes"], w["n_edges"], seed=0, topology=w["topology"])
    return kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w, kg.passage_vid


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C1,C3")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    from hipporag_b200 import Engine
    from hipporag_b200.engine import plan_sweeps
    gpu, limits = card()
    for wl in args.workloads.split(","):
        n, src, dst, w, pv = graph(wl)
        e = Engine(0)
        e.load_graph(n, src, dst, w)
        rng = np.random.default_rng(0)
        R = np.zeros((16, n))
        for q in range(16):          # the shape of a stage-B reset: weighted passages plus a few phrase seeds
            R[q, pv] = 0.05 * rng.random(pv.shape[0])
            R[q, rng.integers(0, n, 5)] += rng.random(5)
        for B in (1, 16):
            for solver in ("ppr", "ppr_f64"):
                fn = (lambda r: e.ppr(r.astype(np.float32))) if solver == "ppr" else (lambda r: e.ppr_f64(r))
                fn(R[:B])                                    # warm-up: allocations, module load
                e.reset_stats()
                t = time.perf_counter()
                for _ in range(args.reps):
                    fn(R[:B])
                wall = (time.perf_counter() - t) * 1e3 / args.reps
                st = e.stats()
                elem = 8 if solver == "ppr_f64" else 4
                h2d, d2h = copy_ms(B * n * elem, args.reps)
                sweeps = st["ppr_sweeps"] / args.reps
                # fp64: every round is one fp32 solve (plan at tol 1e-6) plus one residual sweep
                rounds = sweeps / (plan_sweeps(0.5, 1e-6, 0, B)["fp32_sweeps"] + 1) if solver == "ppr_f64" else None
                print(json.dumps({"workload": wl, "N": n, "B": B, "solver": solver, "ms_per_call": round(wall, 3),
                                  "ms_solve": round(st["ms_ppr"] / args.reps, 3), "ms_h2d": round(h2d, 3),
                                  "ms_d2h": round(d2h, 3), "sweeps_per_call": sweeps, "rounds": rounds,
                                  "error_bound": st["ppr_error_bound"] if solver == "ppr_f64" else None,
                                  "residual": st["ppr_residual"] if solver == "ppr_f64" else None,
                                  "gpu": gpu, "power_limit,max_sm_clock": limits}), flush=True)
        e.close()


if __name__ == "__main__":
    main()
