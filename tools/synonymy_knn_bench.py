"""Cost of the synonymy KNN of add_synonymy_edges per HippoRAG.index() call: today's per-call all-pairs
retrieve_knn(min_score=0.8) against the resident index (knn.retrieve_knn_resident) built once and updated in place.

A synthetic entity matrix at C3 scale (900 k x 768 by default) with planted near-synonym clusters: unit template plus
noise (cosine ~0.9 inside a cluster), cluster sizes chosen so that some rows have no neighbour >= 0.8 but themselves,
some a few, some more than 128 and some more than 512.  Timed, each as host wall time (the call, the dict included)
and device time (the library's stage spans, ms_sim_fact + ms_topk of hrag_get_stats):

* the per-call path, knn.retrieve_knn on a fresh engine (what add_synonymy_edges runs without incremental=True);
* a resident build, then updates after a 1 % append, a 1 % delete and both in one call, and one unchanged call.

After the build and every update the resident lists are compared with a fresh handle's threshold KNN + overflow redo
over the current rows, and must be equal bit for bit.

    python tools/synonymy_knn_bench.py [--rows 900000] [--dim 768] [--json out.json]
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

THR = 0.8


def entities(rng, n, dim, templates, sizes):
    """n rows: len(sizes) clusters of those sizes around `templates`, the rest isotropic noise; unit rows."""
    x = rng.standard_normal((n, dim), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    pos = rng.permutation(n)
    o = 0
    for t, s in zip(templates, sizes):
        idx = pos[o:o + s]
        x[idx] = t + np.float32(0.33) * x[idx]
        o += s
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    return x


def per_call_lists(keys, kmax):
    """A fresh handle's threshold KNN + overflow redo (knn.retrieve_knn's recipe) as [rows, kmax] arrays."""
    from hipporag_b200 import Engine
    e = Engine(0)
    try:
        e.load_embeddings(keys, keys[:1])
        ids, sc, found = e.knn_threshold(0, keys, THR, kmax)
        redo = np.nonzero(found > 512)[0]
        for r0 in range(0, redo.size, 256):
            part = redo[r0:r0 + 256]
            rid, rsc = e.topk_similarity(0, keys[part], int(min(kmax, keys.shape[0])))
            for j, q in enumerate(part):
                keep = rsc[j] >= np.float32(THR)
                ids[q], sc[q] = -1, 0.0
                ids[q, :keep.sum()] = rid[j][keep]
                sc[q, :keep.sum()] = rsc[j][keep]
        return ids, sc, found
    finally:
        e.close()


def device_ms(stats):
    return stats["ms_sim_fact"] + stats["ms_topk"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=900_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--fraction", type=float, default=0.01)
    ap.add_argument("--json", default="")
    args = ap.parse_args()
    import torch
    from hipporag_b200 import Engine, knn
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    out = {"gpu": smi[0] if smi else torch.cuda.get_device_name(0), "rows": args.rows, "dim": args.dim,
           "min_score": THR, "kmax": knn.MAX_CONSUMED}
    print("gpu, power limit:", out["gpu"], flush=True)
    rng = np.random.default_rng(0)
    n_cl = max(4, args.rows // 40)
    sizes = np.r_[[700, 650, 600], [300] * 4, [150] * 8, rng.integers(2, 12, n_cl)]
    templates = rng.standard_normal((sizes.size, args.dim), dtype=np.float32)
    templates /= np.linalg.norm(templates, axis=1, keepdims=True)
    X = entities(rng, args.rows, args.dim, templates, sizes)
    ids = [f"entity-{i}" for i in range(args.rows)]
    nxt = args.rows

    # per-call, as add_synonymy_edges runs it today (a fresh engine per call; its stats read before it closes)
    eng_pc = Engine(0)
    t0 = time.perf_counter()
    ref = knn.retrieve_knn(ids, ids, X, X, k=2047, min_score=THR, engine=eng_pc)
    wall = time.perf_counter() - t0
    out["per_call"] = {"wall_s": wall, "device_ms": device_ms(eng_pc.stats())}
    eng_pc.close()
    print("per-call", json.dumps(out["per_call"]), flush=True)

    eng = Engine(0)
    steps = {}

    def step(name, keys, key_ids, prev):
        # knn.retrieve_knn_resident, timed piece by piece
        eng.reset_stats()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        unit = knn._unit_rows(keys)
        kept_from = knn.classify_keys(prev, list(key_ids))
        t1 = time.perf_counter()
        mode = eng.knn_index_update(unit, kept_from, THR, knn.MAX_CONSUMED)
        t2 = time.perf_counter()
        got_ids, got_sc = eng.knn_index_read()
        res = knn.lists_to_dict(key_ids, got_ids, got_sc)
        t3 = time.perf_counter()
        steps[name] = {"ran": ("built", "updated", "unchanged")[mode], "wall_s": t3 - t0,
                       "wall_normalise_classify_s": t1 - t0, "wall_update_s": t2 - t1, "wall_read_dict_s": t3 - t2,
                       "device_ms": device_ms(eng.stats()), "rows": len(key_ids)}
        want_ids, want_sc, found = per_call_lists(unit, knn.MAX_CONSUMED)
        steps[name]["equal_to_per_call"] = bool(np.array_equal(got_ids, want_ids)
                                                and np.array_equal(got_sc.view(np.uint32), want_sc.view(np.uint32)))
        steps[name]["rows_over_128"] = int((found > 128).sum())
        steps[name]["rows_over_512"] = int((found > 512).sum())
        steps[name]["rows_alone"] = int((found == 1).sum())
        print(name, json.dumps(steps[name]), flush=True)
        return res

    res = step("build", X, ids, None)
    assert res == ref, "resident build differs from the per-call dict"
    del ref, res
    k = int(round(args.fraction * args.rows))
    # 1 % append: half into existing clusters (the big ones included), half noise
    add = entities(rng, k, args.dim, [], [])
    add[: k // 2] = (templates[rng.integers(0, sizes.size, k // 2)]
                     + np.float32(0.33) * rng.standard_normal((k // 2, args.dim), dtype=np.float32) / np.sqrt(args.dim))
    add /= np.linalg.norm(add, axis=1, keepdims=True)
    X2 = np.concatenate([X, add.astype(np.float32)])
    ids2 = ids + [f"entity-{nxt + i}" for i in range(k)]
    nxt += k
    step("append_1pct", X2, ids2, ids)
    keep = np.ones(len(ids2), bool)
    keep[rng.choice(len(ids2), k, replace=False)] = False
    X3, ids3 = np.ascontiguousarray(X2[keep]), [i for i, s in zip(ids2, keep) if s]
    step("delete_1pct", X3, ids3, ids2)
    keep = np.ones(len(ids3), bool)
    keep[rng.choice(len(ids3), k, replace=False)] = False
    add = entities(rng, k, args.dim, templates[:3], [k // 20] * 3)
    X4 = np.concatenate([X3[keep], add])
    ids4 = [i for i, s in zip(ids3, keep) if s] + [f"entity-{nxt + i}" for i in range(k)]
    step("delete_and_append_1pct", X4, ids4, ids3)
    step("unchanged", X4, ids4, ids4)
    out["resident"] = steps
    eng.close()
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
