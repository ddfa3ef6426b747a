"""Graph ingest times on the GPU: Engine.load_graph from host arrays (hrag_load_graph_coo), from CUDA tensors
(hrag_load_graph_coo_device) and load_graph_csr from a float64 CSR (hrag_load_graph_csr_f64), on the C3 and C5 edge
lists of synth.make_kg.  Each time is a host clock around one call that ends in a device synchronise (best of
--reps, after one warm-up load).  For contrast, the host-side scipy build of the same CSR (build_transition_csr).
--profile adds one torch.profiler run of the device-tensor load per graph and prints the device time per kernel.

    python tools/ingest_bench.py [--graphs C3,C5] [--reps 3] [--profile] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GRAPHS = {"C3": (1_000_000, 10_000_000, "uniform"), "C5": (4_000_000, 40_000_000, "powerlaw")}


def timed(fn, reps):
    import torch
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def kernel_times(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            rows[ev.name] = rows.get(ev.name, 0.0) + ev.device_time_total / 1e3
    return dict(sorted(rows.items(), key=lambda kv: -kv[1]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", default="C3,C5")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    import torch
    from hipporag_b200 import Engine, synth
    from hipporag_b200.engine import build_transition_csr
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out = {"gpu": smi[0] if smi else torch.cuda.get_device_name(0), "graphs": {}}
    print("gpu, power limit:", out["gpu"], flush=True)
    for name in args.graphs.split(","):
        n, m, topo = GRAPHS[name]
        kg = synth.make_kg(n, m, seed=0, topology=topo)
        t0 = time.perf_counter()
        row_ptr, col, val = build_transition_csr(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w, dtype=np.float64)
        scipy_s = time.perf_counter() - t0
        src = torch.from_numpy(kg.edge_src).cuda()
        dst = torch.from_numpy(kg.edge_dst).cuda()
        w = torch.from_numpy(kg.edge_w).cuda()
        e = Engine(0)
        host = lambda: e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)   # noqa: E731
        device = lambda: e.load_graph(kg.n_nodes, src, dst, w)                          # noqa: E731
        csr = lambda: e.load_graph_csr(kg.n_nodes, row_ptr, col, val)                  # noqa: E731
        device()                                                                       # warm-up (module load, CUB)
        deg = np.diff(row_ptr)
        res = {"n_nodes": kg.n_nodes, "n_edges": int(kg.n_edges), "nnz": int(col.size), "longest_row": int(deg.max()),
               "coo_host_s": timed(host, args.reps), "coo_device_s": timed(device, args.reps),
               "csr_f64_s": timed(csr, args.reps), "scipy_build_transition_csr_f64_s": scipy_s}
        if args.profile:
            res["device_load_kernels_ms"] = {k: round(v, 3) for k, v in kernel_times(device).items()}
        e.close()
        out["graphs"][name] = res
        print(name, json.dumps(res), flush=True)
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
