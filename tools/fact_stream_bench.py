#!/usr/bin/env python
"""Stage A with the fact planes in pinned host memory (hrag_set_fact_memory) against resident planes.

    python tools/fact_stream_bench.py [--facts 2750000] [--dim 768] [--budget 2e9] [--batches 1024,4096,10000]
                                      [--reps 3] [--big-facts 24000000] [--big-dim 1024] [--skip-big] [--out FILE]

C3 part: one handle with resident planes and one with a --budget ring, loaded from the same seeded rows (generated on
the device and fed to the streamed loader, so no fp32 matrix is held anywhere).  For each batch B the two stage_a calls
alternate, --reps times after a warm-up each; ms per call is the median of host wall time around a call that ends in a
device synchronise (its results are back on the host).  copy_ms is the time the planes alone take to cross the host
link: their bytes over the pinned host-to-device rate, measured with torch copies from a 1 GB pinned buffer in the same
run.  bound_ms = max(copy_ms, resident ms), the least a streamed call could take; identical = ids and scores of the
two handles equal byte for byte.

Big part: one index whose planes exceed the 80 GB of the card (--big-facts x --big-dim x 4 bytes, 98 GB by default),
if the host's available memory holds them with room to spare; otherwise the largest whole-million fact count that fits,
said so in the record.  Reports load time, stage_a q/s at B = 10,000 (one warm-up, then --big-reps calls) and the
device memory the process holds at the end (the CUDA context included).  The pinned planes are the process's own and
go with it.

One JSON line per measurement; every line carries the card's name and power limit, read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402


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


def emit(rec, out):
    line = json.dumps(rec)
    print(line, flush=True)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "a") as f:
            f.write(line + "\n")


def device_chunks(F, dim, seed, rows=1 << 18):
    """(row0, unit rows) chunks of a seeded [F, dim] matrix, generated on the device."""
    import torch
    g = torch.Generator(device="cuda")
    for r0 in range(0, F, rows):
        g.manual_seed(seed * 1_000_003 + r0)
        x = torch.randn((min(rows, F - r0), dim), generator=g, device="cuda", dtype=torch.float32)
        x = (x / x.norm(dim=1, keepdim=True)).contiguous()
        torch.cuda.synchronize()     # the library reads the chunk on its own stream
        yield r0, x


def queries(B, dim, seed):
    import torch
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    x = torch.randn((B, dim), generator=g, device="cuda", dtype=torch.float32)
    return np.ascontiguousarray((x / x.norm(dim=1, keepdim=True)).cpu().numpy())


def load(F, dim, budget, seed):
    from hipporag_b200 import Engine
    e = Engine(0, fact_device_bytes=budget)
    t = time.perf_counter()
    e.load_embeddings_streamed(0, F, dim, device_chunks(F, dim, seed))
    return e, time.perf_counter() - t


def pinned_h2d_rate():
    """Bytes/s of host-to-device copies from a 1 GB pinned buffer (median of 5 runs of 4 copies)."""
    import torch
    n = 1 << 30
    src = torch.empty(n, dtype=torch.uint8, pin_memory=True)
    dst = torch.empty(n, dtype=torch.uint8, device="cuda")
    dst.copy_(src, non_blocking=True)
    torch.cuda.synchronize()
    rates = []
    for _ in range(5):
        t = time.perf_counter()
        for _ in range(4):
            dst.copy_(src, non_blocking=True)
        torch.cuda.synchronize()
        rates.append(4 * n / (time.perf_counter() - t))
    del src, dst
    return float(np.median(rates))


def timed(e, q, k):
    t = time.perf_counter()
    out = e.stage_a(q, k)       # returns host arrays: the call has synchronised
    return (time.perf_counter() - t) * 1e3, out


def c3(args, info, rate):
    F, dim = args.facts, args.dim
    res, t_res = load(F, dim, 0, seed=11)
    host, t_host = load(F, dim, int(args.budget), seed=11)
    plan = host.fact_planes_info()
    emit(dict(info, part="c3_load", facts=F, dim=dim, budget=int(args.budget), resident_load_s=round(t_res, 2),
              host_load_s=round(t_host, 2), **plan), args.out)
    plane_bytes = F * dim * 4
    copy_ms = plane_bytes / rate * 1e3
    for B in [int(b) for b in args.batches.split(",")]:
        q = queries(B, dim, seed=B)
        timed(res, q, 5)
        timed(host, q, 5)
        t_r, t_h, same = [], [], True
        for _ in range(args.reps):
            ms, a = timed(res, q, 5)
            t_r.append(ms)
            ms, b = timed(host, q, 5)
            t_h.append(ms)
            same = same and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
        r_ms, h_ms = float(np.median(t_r)), float(np.median(t_h))
        bound = max(copy_ms, r_ms)
        emit(dict(info, part="c3_stage_a", facts=F, dim=dim, budget=int(args.budget), B=B,
                  resident_ms=round(r_ms, 2), host_ms=round(h_ms, 2), host_over_resident=round(h_ms / r_ms, 3),
                  copy_ms=round(copy_ms, 2), pinned_h2d_GBps=round(rate / 1e9, 2), bound_ms=round(bound, 2),
                  host_over_bound=round(h_ms / bound, 3), identical=bool(same),
                  resident_ms_all=[round(x, 2) for x in t_r], host_ms_all=[round(x, 2) for x in t_h]), args.out)
    res.close()
    host.close()


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
    note = "as asked" if fits == want else (f"host MemAvailable {avail / 1e9:.0f} GB holds {fits} facts, not {want}")
    if fits <= 0:
        emit(dict(info, part="big", skipped=note), args.out)
        return
    free0, total = torch.cuda.mem_get_info()
    e, t_load = load(fits, dim, int(args.budget), seed=13)
    q = queries(10000, dim, seed=7)
    timed(e, q, 5)
    ts = [timed(e, q, 5)[0] for _ in range(args.big_reps)]
    free1, _ = torch.cuda.mem_get_info()
    ms = float(np.median(ts))
    emit(dict(info, part="big", facts=fits, dim=dim, plane_GB=round(fits * dim * 4 / 1e9, 1), note=note,
              budget=int(args.budget), load_s=round(t_load, 1), B=10000, stage_a_ms=round(ms, 1),
              qps=round(10000 / ms * 1e3, 1), copy_ms=round(fits * dim * 4 / rate * 1e3, 1),
              device_used_GB=round((total - free1) / 1e9, 2), device_used_before_GB=round((total - free0) / 1e9, 2),
              **e.fact_planes_info()), args.out)
    e.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--facts", type=int, default=2_750_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--budget", type=float, default=2e9)
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
        sys.exit("fact_stream_bench: no CUDA device")
    info = card()
    rate = pinned_h2d_rate()
    emit(dict(info, part="pinned_h2d", GBps=round(rate / 1e9, 2)), args.out)
    if not args.skip_c3:
        c3(args, info, rate)
    if not args.skip_big:
        big(args, info, rate)


if __name__ == "__main__":
    main()
