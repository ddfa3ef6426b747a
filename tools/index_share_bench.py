#!/usr/bin/env python
"""One index shared between processes on one GPU (hrag_index_export / hrag_index_attach), measured at C3.

    python tools/index_share_bench.py [--nodes 1000000] [--edges 10000000] [--dim 768] [--batch 1024]
                                      [--loop 10] [--workers 1,2,4] [--out FILE]

The owner process loads the index from host arrays (graph as an edge list, tables, fp32 fact and passage rows, so it
keeps the fp32 rows as an index loaded from host memory does) and exports it.  Worker processes (spawned, one Engine
each) attach to it.  Reported, one JSON line each, every line with the card's name and power limit read in this run:

* load: the owner's load time (graph + tables + embeddings, host wall time; every loader returns after its device
  work) against a worker's attach time (hrag_index_attach on a fresh Engine; the Engine's creation, which makes the
  process's CUDA context, is reported apart);
* memory: share_info of the owner and of a worker right after attach (imported_bytes, owned_bytes);
* per_call: stage_a (k = 5) and stage_b of the same --batch queries on the owner and on the worker, alternating, each
  after a warm-up; ms = median of 3 host wall times of calls that end with their results on the host; identical =
  the two handles' outputs equal byte for byte;
* aggregate: 1, 2 and 4 attached workers each running --loop stage_b calls of --batch queries at once; q/s = all
  their queries over the span from the first start to the last end.  The processes time-slice the GPU (no MPS), so
  this is at most about one process's rate; it is reported as measured, not as a speedup.
"""
import argparse
import json
import multiprocessing as mp
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

TIMEOUT = 1800


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


def unit_rows_device(n, dim, seed, rows=1 << 18):
    """[n, dim] fp32 unit rows, generated on the device and returned in host memory."""
    import torch
    out = np.empty((n, dim), np.float32)
    g = torch.Generator(device="cuda")
    for r0 in range(0, n, rows):
        g.manual_seed(seed * 1_000_003 + r0)
        x = torch.randn((min(rows, n - r0), dim), generator=g, device="cuda", dtype=torch.float32)
        out[r0:r0 + x.shape[0]] = (x / x.norm(dim=1, keepdim=True)).cpu().numpy()
    return out


def timed(fn, *args):
    t = time.perf_counter()
    out = fn(*args)
    return (time.perf_counter() - t) * 1e3, out


def stage_calls(eng, inp):
    """The two timed calls on one handle: name -> zero-argument callable returning the outputs."""
    return {"stage_a": lambda: eng.stage_a(inp["qf"], 5),
            "stage_b": lambda: eng.stage_b(inp["qp"], inp["ki"], inp["ks"], None, topk=200)}


def worker(conn):
    """Command loop of one worker process: attach, time one call, loop stage_b, share_info; ("exit",) ends it."""
    from hipporag_b200 import Engine
    eng, inp = None, None
    try:
        while True:
            cmd, *args = conn.recv()
            if cmd == "exit":
                break
            if cmd == "attach":
                t = time.perf_counter()
                eng = Engine(0)
                t1 = time.perf_counter()
                eng.attach(args[0])
                conn.send(((t1 - t) * 1e3, (time.perf_counter() - t1) * 1e3))
            elif cmd == "inputs":
                inp = args[0]
                conn.send(None)
            elif cmd == "time":
                conn.send(timed(stage_calls(eng, inp)[args[0]]))
            elif cmd == "loop":
                fn = stage_calls(eng, inp)["stage_b"]
                fn()                                                    # warm-up
                t0 = time.time()
                for _ in range(args[0]):
                    fn()
                conn.send((t0, time.time()))
            elif cmd == "share_info":
                conn.send(eng.share_info())
    finally:
        if eng is not None:
            eng.close()
        conn.close()


class Worker:
    def __init__(self):
        ctx = mp.get_context("spawn")
        self.conn, theirs = ctx.Pipe()
        self.proc = ctx.Process(target=worker, args=(theirs,), daemon=True)
        self.proc.start()
        theirs.close()

    def send(self, *msg):
        self.conn.send(msg)

    def recv(self):
        if not self.conn.poll(TIMEOUT):
            raise TimeoutError("worker did not answer")
        return self.conn.recv()

    def ask(self, *msg):
        self.send(*msg)
        return self.recv()

    def stop(self):
        try:
            self.conn.send(("exit",))
        except (OSError, ValueError):
            pass
        self.proc.join(TIMEOUT)
        if self.proc.is_alive():
            self.proc.terminate()
            self.proc.join(30)


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "a") as f:
            f.write(line + "\n")


def same(a, b):
    return all(np.asarray(x).tobytes() == np.asarray(y).tobytes() for x, y in zip(a, b))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--nodes", type=int, default=1_000_000)
    ap.add_argument("--edges", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--loop", type=int, default=10)
    ap.add_argument("--workers", default="1,2,4")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    from hipporag_b200 import Engine, synth
    base = dict(card(), nodes=a.nodes, edges=a.edges, dim=a.dim)
    kg = synth.make_kg(a.nodes, a.edges, seed=0)
    fe = unit_rows_device(kg.n_facts, a.dim, seed=1)
    pe = unit_rows_device(kg.n_pass, a.dim, seed=2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, a.batch, seed=3)
    base.update(facts=int(kg.n_facts), passages=int(kg.n_pass))

    owner = Engine(0)
    t = time.perf_counter()
    owner.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    owner.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    owner.load_embeddings(fe, pe)
    load_ms = (time.perf_counter() - t) * 1e3
    del fe, pe
    ki, ks, _ = owner.stage_a(qf, 5)
    inp = dict(qf=qf, qp=qp, ki=ki, ks=ks)
    blob = owner.export_index()
    counts = [int(x) for x in a.workers.split(",")]
    workers = []
    try:
        workers = [Worker() for _ in range(max(counts))]
        ms = [w.ask("attach", blob) for w in workers]
        emit(dict(base, kind="load", owner_load_ms=round(load_ms, 1),
                  worker_engine_create_ms=[round(c, 1) for c, _ in ms], worker_attach_ms=[round(x, 2) for _, x in ms],
                  blob_bytes=len(blob)), a.out)
        for w in workers:
            w.ask("inputs", inp)
        emit(dict(base, kind="memory", owner=owner.share_info(), worker=workers[0].ask("share_info")), a.out)

        mine = stage_calls(owner, inp)
        for name in ("stage_a", "stage_b"):
            want = mine[name]()                                         # warm-up
            _, got = workers[0].ask("time", name)
            ms = {"owner": [], "worker": []}
            for _ in range(3):
                ms["owner"].append(timed(mine[name])[0])
                dt, got = workers[0].ask("time", name)
                ms["worker"].append(dt)
            emit(dict(base, kind="per_call", call=name, batch=a.batch,
                      owner_ms=round(statistics.median(ms["owner"]), 3),
                      worker_ms=round(statistics.median(ms["worker"]), 3), identical=same(got, want)), a.out)

        t0 = time.time()                                                # the owner alone, for reference
        for _ in range(a.loop):
            mine["stage_b"]()
        emit(dict(base, kind="aggregate", processes="owner alone", batch=a.batch,
                  qps=round(a.loop * a.batch / (time.time() - t0), 1)), a.out)
        for n in counts:
            for w in workers[:n]:
                w.send("loop", a.loop)
            spans = [w.recv() for w in workers[:n]]
            span = max(e for _, e in spans) - min(s for s, _ in spans)
            emit(dict(base, kind="aggregate", processes=f"{n} attached worker(s)", batch=a.batch,
                      qps=round(n * a.loop * a.batch / span, 1)), a.out)
    finally:
        for w in workers:
            w.stop()
    owner.unexport()
    owner.close()


if __name__ == "__main__":
    main()
