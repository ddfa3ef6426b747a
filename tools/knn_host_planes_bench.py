"""Cost of the synonymy KNN index with its planes in pinned host memory (hrag_knn_set_memory) against planes on the
device, for the build and the 1 % updates HippoRAG.index() / delete() cause.

Default case: 900 k x 768 unit entities with planted near-synonym clusters (tools/synonymy_knn_bench.py's generator),
threshold 0.8, kmax 128 (knn.MAX_CONSUMED).  Two handles, one with device planes and one at --budget bytes (1 GB),
run the same calls: a build, a 1 % append, a 1 % delete, a 1 % delete + 1 % append in one call, and an unchanged call.
After every call both handles' lists must be equal, bit for bit.

--large: one handle at --budget bytes (2 GB) and d = 1024, with --rows entities; --rows 0 takes the largest whole
million whose fp32 rows and pinned planes (8 KB per entity at d = 1024) fit in 75 % of the host's available memory.

Per call: host wall time of hrag_knn_index_update, device time (the library's stage spans, ms_sim_fact + ms_topk of
hrag_get_stats), the host-to-device bytes the library counted and what those bytes take alone at the pinned
host-to-device rate measured in the same run (a 1 GB pinned buffer).  The card's name and power limit are read in
the same run.

    python tools/knn_host_planes_bench.py [--rows 900000] [--dim 768] [--budget 1e9] [--large] [--json out.json]
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from synonymy_knn_bench import THR, entities  # noqa: E402


def pinned_h2d_gbs():
    import torch
    src = torch.empty(1 << 30, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(1 << 30, dtype=torch.uint8, device="cuda")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(5):
        dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    return 5 * (1 << 30) / (time.perf_counter() - t0) / 1e9


def available_bytes():
    for line in open("/proc/meminfo"):
        if line.startswith("MemAvailable:"):
            return int(line.split()[1]) * 1024
    raise RuntimeError("MemAvailable not found in /proc/meminfo")


def changes(rng, X, dim, templates, fraction):
    """(name, rows, kept_from) of the four updates after a build of X: 1 % append, 1 % delete, both, unchanged."""
    n = X.shape[0]
    k = int(round(fraction * n))
    add = entities(rng, k, dim, templates[:3], [k // 20] * 3)
    X2 = np.concatenate([X, add])
    yield "append_1pct", X2, np.arange(n)
    keep = np.ones(X2.shape[0], bool)
    keep[rng.choice(X2.shape[0], k, replace=False)] = False
    X3 = np.ascontiguousarray(X2[keep])
    yield "delete_1pct", X3, np.flatnonzero(keep)
    del X2
    keep = np.ones(X3.shape[0], bool)
    keep[rng.choice(X3.shape[0], k, replace=False)] = False
    X4 = np.concatenate([X3[keep], entities(rng, k, dim, templates[:3], [k // 20] * 3)])
    yield "delete_and_append_1pct", X4, np.flatnonzero(keep)
    del X3
    yield "unchanged", X4, np.arange(X4.shape[0])


def timed_update(eng, rows, kept_from, kmax):
    eng.reset_stats()
    t0 = time.perf_counter()
    mode = eng.knn_index_update(rows, kept_from, THR, kmax)
    wall = time.perf_counter() - t0
    st = eng.stats()
    return {"ran": ("built", "updated", "unchanged")[mode], "wall_s": wall,
            "device_ms": st["ms_sim_fact"] + st["ms_topk"], "h2d_bytes": int(st["h2d_bytes"])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=900_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--budget", type=float, default=1e9)
    ap.add_argument("--fraction", type=float, default=0.01)
    ap.add_argument("--large", action="store_true")
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    import torch
    from hipporag_b200 import Engine, knn
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    kmax = knn.MAX_CONSUMED
    avail = available_bytes()
    by_memory = int(0.75 * avail // (8 * args.dim)) // 1_000_000 * 1_000_000
    if args.large and args.rows == 0:
        args.rows = by_memory
    budget = int(args.budget)
    gbs = pinned_h2d_gbs()
    out = {"gpu": smi[0] if smi else torch.cuda.get_device_name(0), "rows": args.rows, "dim": args.dim,
           "min_score": THR, "kmax": kmax, "budget_bytes": budget, "host_available_bytes": avail,
           "rows_by_memory_rule": by_memory,
           "plane_bytes": args.rows * args.dim * 4, "pinned_h2d_gbs": gbs}
    print(json.dumps(out), flush=True)
    rng = np.random.default_rng(0)
    n_cl = max(4, args.rows // 40)
    sizes = np.r_[[700, 650, 600], [300] * 4, [150] * 8, rng.integers(2, 12, n_cl)]
    templates = rng.standard_normal((sizes.size, args.dim), dtype=np.float32)
    templates /= np.linalg.norm(templates, axis=1, keepdims=True)
    X = entities(rng, args.rows, args.dim, templates, sizes)

    host = Engine(0)
    host.knn_set_memory(budget)
    dev = None if args.large else Engine(0)
    steps = {}
    for name, rows, kept_from in [("build", X, None)] + list(changes(rng, X, args.dim, templates, args.fraction)):
        s = {"rows": rows.shape[0], "host_planes": timed_update(host, rows, kept_from, kmax)}
        s["host_planes"]["copy_alone_ms"] = s["host_planes"]["h2d_bytes"] / gbs / 1e6
        s["planes_info"] = host.knn_planes_info()
        if dev is not None:
            s["device_planes"] = timed_update(dev, rows, kept_from, kmax)
            a, b = host.knn_index_read(), dev.knn_index_read()
            s["lists_equal"] = bool(np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32),
                                                                                   b[1].view(np.uint32)))
            del a, b
        steps[name] = s
        print(name, json.dumps(s), flush=True)
    out["steps"] = steps
    host.close()
    if dev is not None:
        dev.close()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
