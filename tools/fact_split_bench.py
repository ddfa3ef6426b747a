#!/usr/bin/env python
"""Stage A with the hi fact plane resident and the lo plane in pinned host memory (HRAG_FACT_LO_ON_HOST) against
resident planes and against both planes in host memory (hrag_set_fact_memory alone).

    python tools/fact_split_bench.py [--facts 2750000] [--dim 768] [--batches 1024,4096,10000] [--reps 3]
                                     [--big-facts 24000000] [--big-dim 1024] [--skip-big] [--out FILE]

C3 part: four handles loaded from the same seeded rows (generated on the device and fed to the streamed loader):
resident; lo on the host at a budget of the hi plane + 1 GB; both planes on the host at that same budget; both planes
on the host at 2 GB (the DESIGN.md section 7e row).  For each batch B the four stage_a calls (k = 5) alternate, --reps
times after a warm-up each; ms per call is the median of host wall time around a call whose results are back on the
host.  Per call of the lo-on-host handle: the lo bytes its gathers read over PCIe (h2d_bytes less the query upload),
the rows that is (a row staged by two 128-query m-tiles of a chunk counts twice), and its fallbacks; identical = ids,
scores and n_valid of every handle equal the resident ones byte for byte.

Big part: one index of --big-dim columns sized by section 7e's rule (--big-facts, or the largest whole-million count
whose planes take at most 75 % of the host's available memory), at a budget of its hi plane + 1 GB: lo on the host,
then both planes on the host, one after the other (both pinned sets would not fit at once), stage_a at B = 10,000 (one
warm-up, then --big-reps calls).  Each record carries the stage-A query chunk the screen ran at.

One JSON line per measurement; every line carries the card's name and power limit, read in the same run.
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from fact_stream_bench import card, device_chunks, emit, pinned_h2d_rate, queries  # noqa: E402

GB = 1 << 30


def load(F, dim, budget, lo_on_host, seed):
    from hipporag_b200 import Engine
    e = Engine(0, fact_device_bytes=budget, fact_lo_on_host=lo_on_host)
    t = time.perf_counter()
    e.load_embeddings_streamed(0, F, dim, device_chunks(F, dim, seed))
    return e, time.perf_counter() - t


def call(e, q, k=5):
    """(ms, outputs, fallbacks, h2d bytes) of one stage_a call."""
    e.reset_stats()
    t = time.perf_counter()
    out = e.stage_a(q, k)       # returns host arrays: the call has synchronised
    ms = (time.perf_counter() - t) * 1e3
    st = e.stats()
    return ms, out, int(st["stage_a_fallbacks"]), int(st["h2d_bytes"])


def screen_chunk(F):
    """The screen's query chunk under HRAG_FACT_LO_ON_HOST (fact_stream.cu lo_host_chunk)."""
    per_query = 88 * -(-F // 256)
    return min(1024, max(128, GB // per_query // 128 * 128))


def c3(args, info, rate):
    F, dim = args.facts, args.dim
    hi = F * dim * 2
    plans = [("resident", 0, False), ("lo_on_host", hi + GB, True), ("host_planes", hi + GB, False),
             ("host_planes_2GB", 2 * 10**9, False)]
    engines = {}
    for name, budget, lo in plans:
        engines[name], t_load = load(F, dim, budget, lo, seed=11)
        emit(dict(info, part="c3_load", handle=name, facts=F, dim=dim, budget=budget, load_s=round(t_load, 2),
                  **engines[name].fact_planes_info()), args.out)
    for B in [int(b) for b in args.batches.split(",")]:
        q = queries(B, dim, seed=B)
        q_bytes = q.nbytes
        for e in engines.values():
            call(e, q)
        times = {name: [] for name in engines}
        lo_bytes, fallbacks, same = [], [], True
        for _ in range(args.reps):
            ref = None
            for name, e in engines.items():
                ms, out, fb, h2d = call(e, q)
                times[name].append(ms)
                if name == "resident":
                    ref = out
                else:
                    same = same and all(a.tobytes() == b.tobytes() for a, b in zip(out, ref))
                if name == "lo_on_host":
                    lo_bytes.append(h2d - q_bytes)
                    fallbacks.append(fb)
        med = {name: round(float(np.median(t)), 2) for name, t in times.items()}
        emit(dict(info, part="c3_stage_a", facts=F, dim=dim, B=B, k=5, ms=med,
                  lo_on_host_over_resident=round(med["lo_on_host"] / med["resident"], 3),
                  lo_gathered_MB=round(float(np.median(lo_bytes)) / 1e6, 1),
                  lo_rows_gathered=int(np.median(lo_bytes)) // (2 * dim), fallbacks=fallbacks,
                  screen_chunk=screen_chunk(F), pinned_h2d_GBps=round(rate / 1e9, 2), identical=bool(same),
                  ms_all={name: [round(x, 2) for x in t] for name, t in times.items()}), args.out)
    for e in engines.values():
        e.close()


def big(args, info, rate):
    import torch
    dim = args.big_dim
    avail = 0
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                avail = int(line.split()[1]) * 1024
    want = args.big_facts
    fits = min(want, int(0.75 * avail) // (dim * 4) // 1_000_000 * 1_000_000)
    note = "as asked" if fits == want else f"host MemAvailable {avail / 1e9:.0f} GB holds {fits} facts, not {want}"
    if fits <= 0:
        emit(dict(info, part="big", skipped=note), args.out)
        return
    budget = fits * dim * 2 + GB
    q = queries(10000, dim, seed=7)
    ref = None
    for name, lo in (("lo_on_host", True), ("host_planes", False)):
        free0, total = torch.cuda.mem_get_info()
        e, t_load = load(fits, dim, budget, lo, seed=13)
        call(e, q)
        runs = [call(e, q) for _ in range(args.big_reps)]
        free1, _ = torch.cuda.mem_get_info()
        ms = float(np.median([r[0] for r in runs]))
        out = runs[-1][1]
        same = None if ref is None else all(a.tobytes() == b.tobytes() for a, b in zip(out, ref))
        ref = out if ref is None else ref
        rec = dict(info, part="big", handle=name, facts=fits, dim=dim, plane_GB=round(fits * dim * 4 / 1e9, 1),
                   note=note, budget=budget, load_s=round(t_load, 1), B=10000, k=5, stage_a_ms=round(ms, 1),
                   qps=round(10000 / ms * 1e3, 1), fallbacks=[r[2] for r in runs],
                   device_used_GB=round((total - free1) / 1e9, 2), device_used_before_GB=round((total - free0) / 1e9, 2),
                   **e.fact_planes_info())
        if lo:
            rec.update(screen_chunk=screen_chunk(fits),
                       lo_gathered_GB=round(float(np.median([r[3] for r in runs]) - q.nbytes) / 1e9, 2))
        else:
            rec.update(identical_to_lo_on_host=same)
        emit(rec, args.out)
        e.close()
        del e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--facts", type=int, default=2_750_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batches", default="1024,4096,10000")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--big-facts", type=int, default=24_000_000)
    ap.add_argument("--big-dim", type=int, default=1024)
    ap.add_argument("--big-reps", type=int, default=2)
    ap.add_argument("--skip-big", action="store_true")
    ap.add_argument("--skip-c3", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("fact_split_bench: no CUDA device")
    info = card()
    rate = pinned_h2d_rate()
    emit(dict(info, part="pinned_h2d", GBps=round(rate / 1e9, 2)), args.out)
    if not args.skip_c3:
        c3(args, info, rate)
    if not args.skip_big:
        big(args, info, rate)


if __name__ == "__main__":
    main()
