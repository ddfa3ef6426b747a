"""The graph planes built on the device, byte for byte, against a numpy restatement of the sequential host build.

The restatement symmetrises the edge list (entry 2i = (a -> b), 2i + 1 = (b -> a), weights not > 0 dropped), orders
the entries by (row, col) with a stable sort, sums each run of parallel edges in input order and each row's merged
weights in column order -- by iterating along the runs / rows while vectorising across them, which is exactly the
sequential order -- divides in float64 and packs the fp32 planes with round-to-nearest.  Every loader (host and device
COO, fp64 and fp32 CSR) must give its planes bit for bit, and therefore the same solves.
"""
import functools
import os
import socket

import numpy as np
import pytest

DIM = 64
LOADERS = ("coo_host", "coo_device", "csr_f64", "csr_f32")


# ----------------------------------------------------------------------------- the restatement
def _sequential_sums(values, starts, lens):
    """out[i] = ((0.0 + values[starts[i]]) + values[starts[i] + 1]) + ... over lens[i] terms, for every i at once."""
    out = np.zeros(len(starts))
    if len(starts) == 0:
        return out
    order = np.argsort(-lens, kind="stable")
    st, ln = starts[order], lens[order]
    acc = np.zeros(len(starts))
    neg = -ln                                          # ascending
    for j in range(int(ln[0])):
        c = int(np.searchsorted(neg, -j, side="left"))   # the runs longer than j are a prefix
        acc[:c] += values[st[:c] + j]
    out[order] = acc
    return out


def restate_csr(n, src, dst, w):
    """(row_ptr int64 [n + 1], col int32, val float64) of P = W D^-1 as the sequential host build makes it."""
    src, dst, w = (np.asarray(src, np.int64), np.asarray(dst, np.int64), np.asarray(w, np.float64))
    keep = w > 0
    a, b, x = src[keep], dst[keep], w[keep]
    rows = np.empty(2 * a.size, np.int64)
    cols = np.empty(2 * a.size, np.int64)
    rows[0::2], rows[1::2], cols[0::2], cols[1::2] = a, b, b, a
    key = (rows << 32) | cols
    order = np.argsort(key, kind="stable")
    key, ww = key[order], np.repeat(x, 2)[order]
    starts = np.flatnonzero(np.r_[True, key[1:] != key[:-1]]) if key.size else np.zeros(0, np.int64)
    wsum = _sequential_sums(ww, starts, np.diff(np.r_[starts, key.size]))
    urow, col = key[starts] >> 32, (key[starts] & 0xffffffff).astype(np.int32)
    row_ptr = np.zeros(n + 1, np.int64)
    row_ptr[1:] = np.cumsum(np.bincount(urow, minlength=n))
    strength = _sequential_sums(wsum, row_ptr[:-1], np.diff(row_ptr))
    return row_ptr, col, wsum / strength[col] if col.size else wsum


def planes_of(row_ptr, col, val, lo=0, hi=None, f64=True):
    """The planes of rows [lo, hi) of a CSR, as hrag_debug_graph returns them."""
    hi = len(row_ptr) - 1 if hi is None else hi
    a, b = int(row_ptr[lo]), int(row_ptr[hi])
    rp = (row_ptr[lo:hi + 1] - a).astype(np.int32)
    v = val[a:b]
    vhi = v.astype(np.float32)
    out = dict(row_ptr=rp, cv=np.stack([col[a:b].astype(np.int32), vhi.view(np.int32)], axis=1),
               val_lo=(v - vhi.astype(np.float64)).astype(np.float32) if f64 else np.zeros(0, np.float32))
    lens = np.diff(rp)
    n_rows = len(lens)
    out["row_order"] = np.lexsort((-lens, np.arange(n_rows) // 64)).astype(np.int32)   # stable within each block
    long_rows = np.flatnonzero(lens > 256).astype(np.int32)
    segs = [(r, s, min(int(rp[r + 1]), s + 256), 0) for r in long_rows for s in range(int(rp[r]), int(rp[r + 1]), 256)]
    nseg = (lens[long_rows] + 255) // 256
    out["long_rows"] = long_rows
    out["long_seg_ptr"] = np.r_[0, np.cumsum(nseg)].astype(np.int32) if long_rows.size else np.zeros(0, np.int32)
    out["segs"] = np.array(segs, np.int32).reshape(-1, 4)
    return out


# ----------------------------------------------------------------------------- graphs
def _row_lengths_graph():
    """Vertices 0..K-1 are centres whose row lengths are exactly 0-9, 255-257, 511-513, a hub of 5,000 and 70 more
    long rows (> 64 long rows in all); their neighbours are distinct leaves, so a centre's row holds each once."""
    rng = np.random.default_rng(11)
    degs = list(range(10)) + [255, 256, 257, 511, 512, 513, 5000] + list(range(300, 370))
    n = 6000
    k = len(degs)
    src, dst = [], []
    for c, d in enumerate(degs):
        leaves = rng.choice(np.arange(k, n), d, replace=False)
        src.append(np.full(d, c))
        dst.append(leaves)
    src, dst = np.concatenate(src), np.concatenate(dst)
    flip = rng.random(src.size) < 0.5                  # either orientation
    src, dst = np.where(flip, dst, src), np.where(flip, src, dst)
    return n, src, dst, rng.uniform(0.1, 3.0, src.size)


def _edge_cases_graph():
    """Self-loops, (u, v) given with (v, u), runs of parallel edges whose sums show the order, zero, negative and NaN
    weights, isolated vertices (the tail of the id range has no edge)."""
    t = 2.0 ** -53
    e = [(0, 1, 1.0), (0, 1, t), (1, 0, t),           # (1 + t) + t = 1 in this order; 1 + 2t the other way
         (2, 3, t), (3, 2, t), (2, 3, 1.0),           # (t + t) + 1 = 1 + 2t
         (1, 10, 1.0), (3, 11, 1.0),                  # so that the strengths of 1 and 3 do not cancel those sums
         (4, 4, 0.75), (4, 4, 0.25), (4, 5, 1.5),     # self-loops count twice
         (5, 6, 0.0), (6, 7, -1.0), (7, 8, np.nan), (8, 9, 2.0), (9, 8, 3.0), (5, 9, 1e-300), (5, 9, 1e300)]
    rng = np.random.default_rng(5)
    n = 200
    src = np.r_[[a for a, _, _ in e], rng.integers(10, 150, 400)]
    dst = np.r_[[b for _, b, _ in e], rng.integers(10, 150, 400)]
    w = np.r_[[x for _, _, x in e], rng.choice([1.0, t, 0.5, 3.0, -2.0, 0.0], 400)]
    return n, src, dst, w


def _random_graph(n, m, seed):
    rng = np.random.default_rng(seed)
    return n, rng.integers(0, n, m), rng.integers(0, n, m), rng.choice([0.5, 1.0, 2.0 ** -30, 7.0, -1.0], m)


@functools.lru_cache(maxsize=None)
def graph(name):
    if name == "row_lengths":
        return _row_lengths_graph()
    if name == "edge_cases":
        return _edge_cases_graph()
    if name == "all_dropped":
        return 50, np.arange(40), np.arange(1, 41), np.r_[np.zeros(20), -np.ones(10), np.full(10, np.nan)]
    if name == "no_edges":
        return 7, np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0)
    if name.startswith("n"):
        n = int(name[1:])
        return _random_graph(n, 5 * n + 3, n)
    if name == "powerlaw":
        from hipporag_b200 import synth
        kg = synth.make_kg(200_000, 2_000_000, seed=3, topology="powerlaw")
        return kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w
    raise KeyError(name)


GRAPHS = ["row_lengths", "edge_cases", "all_dropped", "no_edges", "n1", "n63", "n64", "n65", "n4133", "powerlaw"]


# ----------------------------------------------------------------------------- loading
def load(e, loader, n, src, dst, w):
    import torch
    if loader == "coo_host":
        e.load_graph(n, src, dst, w)
    elif loader == "coo_device":
        dev = f"cuda:{e.device}"
        e.load_graph(n, torch.tensor(np.asarray(src, np.int32), device=dev),
                     torch.tensor(np.asarray(dst, np.int32), device=dev), torch.tensor(np.asarray(w, np.float64), device=dev))
    else:
        row_ptr, col, val = restate_csr(n, src, dst, w)
        e.load_graph_csr(n, row_ptr, col, val if loader == "csr_f64" else val.astype(np.float32))


def got_planes(e):
    return {p: e.debug_graph(p) for p in e.GRAPH_PLANES}


def assert_planes_equal(got, want, what):
    for p, v in want.items():
        g = got[p]
        assert g.dtype == v.dtype and g.shape == v.shape, (what, p, g.shape, v.shape)
        assert np.array_equal(g.view(np.uint8), v.view(np.uint8)), f"{what}: plane {p} differs"


@pytest.fixture(scope="module")
def hb():
    import hipporag_b200
    return hipporag_b200


@pytest.fixture(scope="module")
def engine(hb):
    e = hb.Engine(0)
    yield e
    e.close()


# ----------------------------------------------------------------------------- CPU: the restatement itself
def test_restatement_matches_transition_csr():
    """The restatement's structure equals build_transition_csr's and its values agree to rounding (the scipy build
    sums in another order); the order-sensitive runs of the edge-case graph come out as the sequential order gives."""
    from hipporag_b200.engine import build_transition_csr
    for name in ("row_lengths", "edge_cases", "n65", "all_dropped"):
        n, src, dst, w = graph(name)
        row_ptr, col, val = restate_csr(n, src, dst, w)
        rp2, col2, val2 = build_transition_csr(n, src, dst, w, dtype=np.float64)
        assert np.array_equal(row_ptr, rp2) and np.array_equal(col, col2), name
        np.testing.assert_allclose(val, val2, rtol=1e-14, err_msg=name)
    n, src, dst, w = graph("edge_cases")
    row_ptr, col, val = restate_csr(n, src, dst, w)
    t = 2.0 ** -53
    assert col[row_ptr[0]] == 1 and val[row_ptr[0]] == 0.5           # W01 = (1 + t) + t = 1, strength of 1 = 1 + 1
    assert col[row_ptr[2]] == 3 and val[row_ptr[2]] == 0.5 + t       # W23 = (t + t) + 1, strength of 3 = fl(2 + 2t) = 2
    lens = np.diff(planes_of(*restate_csr(*graph("row_lengths")))["row_ptr"])
    assert list(lens[:17]) == list(range(10)) + [255, 256, 257, 511, 512, 513, 5000]


# ----------------------------------------------------------------------------- GPU: planes
@pytest.mark.gpu
@pytest.mark.parametrize("name", GRAPHS)
def test_planes_equal_restatement(engine, name):
    n, src, dst, w = graph(name)
    row_ptr, col, val = restate_csr(n, src, dst, w)
    for loader in LOADERS:
        load(engine, loader, n, src, dst, w)
        assert_planes_equal(got_planes(engine), planes_of(row_ptr, col, val, f64=loader != "csr_f32"),
                            f"{name} via {loader}")


# ----------------------------------------------------------------------------- GPU: solves
def _kg_with_hub(seed, hub_deg=600):
    from hipporag_b200 import synth
    kg = synth.make_kg(4000, 40000, seed=seed)
    rng = np.random.default_rng(seed)
    hub = rng.choice(np.arange(1, kg.n_nodes), hub_deg, replace=False).astype(np.int32)
    src = np.concatenate([kg.edge_src, np.zeros(hub_deg, np.int32)])
    dst = np.concatenate([kg.edge_dst, hub])
    w = np.concatenate([kg.edge_w, rng.uniform(0.5, 2.0, hub_deg)])
    return kg, src, dst, w


def _resets(n, b, seed):
    rng = np.random.default_rng(seed)
    r = np.zeros((b, n), np.float32)
    for i in range(b):
        r[i, rng.choice(n, 5, replace=False)] = rng.uniform(0.1, 1.0, 5)
    return r


def _engine(hb, loader, kg, src, dst, w):
    from hipporag_b200 import synth
    e = hb.Engine(0)
    load(e, loader, kg.n_nodes, src, dst, w)
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    e.load_embeddings(synth.unit_rows(kg.n_facts, DIM, seed=1), synth.unit_rows(kg.n_pass, DIM, seed=2))
    return e


def _results(e, kg, f64=True):
    from hipporag_b200 import synth
    fe = synth.unit_rows(kg.n_facts, DIM, seed=1)
    pe = synth.unit_rows(kg.n_pass, DIM, seed=2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 40, seed=3)
    idx, score, _ = e.stage_a(qf, k=5)
    ids, scores = e.stage_b(qp, idx, score)
    out = dict(fp32=e.ppr(_resets(kg.n_nodes, 4, 4)), mixed=e.ppr(_resets(kg.n_nodes, 40, 5)), stage_b_ids=ids,
               stage_b_scores=scores)
    if f64:
        out["f64"] = e.ppr_f64(_resets(kg.n_nodes, 4, 6).astype(np.float64))
    return out


def _assert_same(got, want, what):
    for k in got:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, (what, k)
        assert np.array_equal(got[k].view(np.uint8), want[k].view(np.uint8)), f"{what}: {k} differs"


@pytest.mark.gpu
def test_solves_identical_across_loaders(hb):
    kg, src, dst, w = _kg_with_hub(7)
    e = _engine(hb, "coo_host", kg, src, dst, w)
    want = _results(e, kg)
    e.close()
    for loader in LOADERS[1:]:
        e = _engine(hb, loader, kg, src, dst, w)
        _assert_same(_results(e, kg, f64=loader != "csr_f32"), want, loader)
        e.close()


# ----------------------------------------------------------------------------- GPU: the device entry
@pytest.mark.gpu
def test_device_entry_rejections_keep_the_handle(hb):
    import torch
    kg, src, dst, w = _kg_with_hub(7)
    e = _engine(hb, "coo_device", kg, src, dst, w)
    want = _results(e, kg)
    want_planes = got_planes(e)
    n = kg.n_nodes
    d_src = torch.tensor(src, dtype=torch.int32, device="cuda:0")
    d_dst = torch.tensor(dst, dtype=torch.int32, device="cuda:0")
    d_w = torch.tensor(w, dtype=torch.float64, device="cuda:0")
    too_big, negative = d_dst.clone(), d_src.clone()
    too_big[len(too_big) // 2] = n
    negative[-1] = -1
    library = [
        ("endpoint = N", lambda: e.load_graph(n, d_src, too_big, d_w), "edge endpoint out of range"),
        ("endpoint = -1", lambda: e.load_graph(n, negative, d_dst, d_w), "edge endpoint out of range"),
        ("N = 0", lambda: e.load_graph(0, d_src, d_dst, d_w), "sizes out of range"),
        ("N = 2^30", lambda: e.load_graph(1 << 30, d_src, d_dst, d_w), "sizes out of range"),
    ]
    for what, call, msg in library:
        with pytest.raises(hb.HragError, match=msg):
            call()
        _assert_same(_results(e, kg), want, f"after a rejected load ({what})")
    python = [
        ("int64 src", lambda: e.load_graph(n, d_src.long(), d_dst, d_w)),
        ("float32 weights", lambda: e.load_graph(n, d_src, d_dst, d_w.float())),
        ("non-contiguous", lambda: e.load_graph(n, torch.stack([d_src, d_src], 1)[:, 0], d_dst, d_w)),
        ("CPU tensor", lambda: e.load_graph(n, d_src.cpu(), d_dst, d_w)),
        ("numpy mixed with tensors", lambda: e.load_graph(n, src, d_dst, d_w)),
        ("mismatched lengths", lambda: e.load_graph(n, d_src, d_dst[:-1], d_w)),
    ]
    for what, call in python:
        with pytest.raises(ValueError):
            call()
        _assert_same(_results(e, kg), want, f"after a rejected load ({what})")
    assert_planes_equal(got_planes(e), want_planes, "after the rejections")
    e.close()


@pytest.mark.gpu
def test_device_reload_invalidates_captured_solves(hb):
    import torch
    kg, src, dst, w = _kg_with_hub(7)
    e = _engine(hb, "coo_device", kg, src, dst, w)
    resets = _resets(kg.n_nodes, 40, 8)
    first = e.ppr(resets)                            # captures the mixed solve for this buffer set and plan
    kg2, src2, dst2, w2 = _kg_with_hub(8, hub_deg=900)
    assert kg2.n_nodes == kg.n_nodes
    e.load_graph(kg2.n_nodes, torch.tensor(src2, device="cuda:0"), torch.tensor(dst2, device="cuda:0"),
                 torch.tensor(w2, device="cuda:0"))
    got = e.ppr(resets)
    fresh = _engine(hb, "coo_host", kg2, src2, dst2, w2)
    want = fresh.ppr(resets)
    assert not np.array_equal(first, want)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    fresh.close()
    e.close()


# ----------------------------------------------------------------------------- GPU: node-range sharding
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _sharded_worker(rank, world, port, out_dir):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)      # only carries the NCCL id
    from hipporag_b200 import Engine
    n, src, dst, w = graph("powerlaw")
    ids = [Engine.new_comm_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    e = Engine(rank, shard_mode=1)
    e.init_comm(ids[0], rank, world)
    for loader in ("coo_host", "coo_device"):
        load(e, loader, n, src, dst, w)
        np.savez(os.path.join(out_dir, f"{loader}_{rank}.npz"), **got_planes(e))
    dist.barrier()
    e.close()
    dist.destroy_process_group()


@pytest.mark.gpu
def test_sharded_device_entry_matches_host_entry(tmp_path):
    """Each rank of a 2-GPU node-range-sharded handle gets the same rows and planes from both COO entries: the rows of
    the work-balanced partition of the full graph."""
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from hipporag_b200.engine import balanced_row_bounds
    mp.spawn(_sharded_worker, args=(2, _free_port(), str(tmp_path)), nprocs=2, join=True)
    row_ptr, col, val = restate_csr(*graph("powerlaw"))
    bounds = balanced_row_bounds(row_ptr, 2)
    for rank in range(2):
        want = planes_of(row_ptr, col, val, int(bounds[rank]), int(bounds[rank + 1]))
        for loader in ("coo_host", "coo_device"):
            got = dict(np.load(tmp_path / f"{loader}_{rank}.npz"))
            assert_planes_equal(got, want, f"rank {rank} via {loader}")
