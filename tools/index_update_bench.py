"""Cost of an in-place index update against a full reload, on the C3 index of synth.make_kg (1 M vertices, 10 M edges,
dim 768).  The index is split into a base and the last 1 % of its passages (vertex ids at the end of the range) with
every edge incident to them and every fact planted on them (moved to the end of the fact rows).  Timed:

* a full reload of the whole index on a mutable handle: the graph from CUDA tensors and from host arrays, the tables,
  the embeddings (host arrays), each a host clock around calls that end in a device synchronise;
* Engine.append of the 1 % and Engine.delete of it again, each as device time (CUDA events on hrag_stream) and host
  wall time, best of --reps.

    python tools/index_update_bench.py [--config C3] [--reps 3] [--json out.json]
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


def best_wall(fn, reps):
    import torch
    best = float("inf")
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="C3")
    ap.add_argument("--fraction", type=float, default=0.01)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    import torch
    from hipporag_b200 import Engine, synth
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out = {"gpu": smi[0] if smi else torch.cuda.get_device_name(0), "config": args.config}
    print("gpu, power limit:", out["gpu"], flush=True)
    n, m, dim = synth.CONFIGS[args.config][:3]
    kg = synth.make_kg(n, m, seed=0, topology=synth.CONFIGS[args.config][4])
    fe = synth.unit_rows(kg.n_facts, dim, seed=1)
    pe = synth.unit_rows(kg.n_pass, dim, seed=2)

    # the last k passages are the last k vertices; their facts go to the end of the fact rows
    k = max(1, int(round(args.fraction * kg.n_pass)))
    N, N0 = kg.n_nodes, kg.n_nodes - k
    tail_f = kg.fact_passage >= kg.n_pass - k
    forder = np.r_[np.flatnonzero(~tail_f), np.flatnonzero(tail_f)]
    fs, fo, fe = kg.fact_subj_vid[forder], kg.fact_obj_vid[forder], np.ascontiguousarray(fe[forder])
    F0 = int((~tail_f).sum())
    tail_e = (kg.edge_src >= N0) | (kg.edge_dst >= N0)
    eorder = np.r_[np.flatnonzero(~tail_e), np.flatnonzero(tail_e)]
    src, dst, w = kg.edge_src[eorder], kg.edge_dst[eorder], kg.edge_w[eorder]
    E0 = int((~tail_e).sum())
    P0 = kg.n_pass - k
    cc0 = kg.ent_chunk_count                              # kept as given for the base and the whole index
    out.update(n_nodes=N, n_edges=int(src.size), n_facts=int(fs.size), n_passages=int(kg.n_pass), dim=dim,
               appended={"vertices": k, "passages": k, "edges": int(src.size - E0), "facts": int(fs.size - F0)})

    e = Engine(0, mutable=True)
    d_src, d_dst, d_w = (torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (src, dst, w))
    e.load_graph(N, d_src, d_dst, d_w)                     # warm-up (module load, CUB)
    out["reload_s"] = {
        "graph_device": best_wall(lambda: e.load_graph(N, d_src, d_dst, d_w), args.reps),
        "graph_host": best_wall(lambda: e.load_graph(N, src, dst, w), args.reps),
        "tables": best_wall(lambda: e.load_tables(kg.passage_vid, fs, fo, kg.ent_chunk_count), args.reps),
        "embeddings": best_wall(lambda: e.load_embeddings(fe, pe), args.reps),
    }
    out["reload_s"]["total_graph_host"] = (out["reload_s"]["graph_host"] + out["reload_s"]["tables"]
                                           + out["reload_s"]["embeddings"])
    print("reload", json.dumps(out["reload_s"]), flush=True)
    # the base: the same index without the last k passages
    e.load_graph(N0, src[:E0], dst[:E0], w[:E0])
    e.load_tables(kg.passage_vid[:P0], fs[:F0], fo[:F0], cc0[:N0])
    e.load_embeddings(fe[:F0], pe[:P0])
    e.reserve(nodes=N, edges=int(src.size), facts=int(fs.size), passages=int(kg.n_pass))
    stream = torch.cuda.ExternalStream(e.stream_ptr)
    new_nodes = np.arange(N0, N, dtype=np.int32)
    new_facts = np.arange(F0, fs.size, dtype=np.int32)

    def append():
        e.append(k, src[E0:], dst[E0:], w[E0:], kg.passage_vid[P0:], fs[F0:], fo[F0:], cc0, fe[F0:], pe[P0:])

    def delete():
        e.delete(new_nodes, new_facts, cc0[:N0])

    res = {name: {"device_ms": float("inf"), "wall_ms": float("inf")} for name in ("append", "delete")}
    for rnd in range(args.reps + 1):                       # round 0 warms up
        for name, fn in (("append", append), ("delete", delete)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            a.record(stream)
            fn()
            b.record(stream)
            torch.cuda.synchronize()
            wall = (time.perf_counter() - t0) * 1e3
            if rnd:
                res[name]["device_ms"] = min(res[name]["device_ms"], a.elapsed_time(b))
                res[name]["wall_ms"] = min(res[name]["wall_ms"], wall)
    out["update_ms"] = res
    print("update", json.dumps(res), flush=True)
    e.close()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
