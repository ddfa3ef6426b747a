"""world_size-2 CPU (gloo) test of the node-range sharding HOST logic: the row partition and CSR
slicing `Engine.load_graph_csr` uses, driven through the same exchange pattern as the GPU path
(every rank sweeps its own rows, one all-gather per sweep) with numpy standing in for the kernel."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import ppr


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, n, src, dst, w, R, out_path):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hipporag_b200.engine import build_transition_csr, shard_rows, slice_csr_rows
    import scipy.sparse as sp
    row_ptr, col, val = build_transition_csr(n, src, dst, w)
    lo, hi = shard_rows(n, rank, world)
    rp, c, v = slice_csr_rows(row_ptr, col, val, lo, hi)
    P_local = sp.csr_matrix((v.astype(np.float64), c, rp), shape=(hi - lo, n))
    chunk = -(-n // world)
    V = np.zeros((chunk * world, R.shape[1]))
    V[:n] = R
    X = V.copy()
    for _ in range(60):                                  # z <- a P z + v on the owned rows, then all-gather
        y_local = np.zeros((chunk, R.shape[1]))
        y_local[:hi - lo] = 0.5 * (P_local @ X[:n]) + V[lo:hi]
        parts = [torch.zeros(chunk, R.shape[1], dtype=torch.float64) for _ in range(world)]
        dist.all_gather(parts, torch.from_numpy(y_local))
        X = torch.cat(parts).numpy()
    if rank == 0:
        Z = X[:n]
        np.save(out_path, Z / Z.sum(axis=0, keepdims=True))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("n", [101, 256])
def test_two_rank_sharded_sweeps_match_oracle(tmp_path, n):
    rng = np.random.default_rng(n)
    src, dst = rng.integers(0, n - 2, 6 * n), rng.integers(0, n - 2, 6 * n)
    keep = src != dst
    src, dst = src[keep], dst[keep]
    w = rng.random(src.shape[0]) + 0.2
    R = rng.random((n, 3)) * (rng.random((n, 3)) < 0.3)
    R[0] += 0.1
    out = str(tmp_path / "pi.npy")
    mp.spawn(_worker, args=(2, _free_port(), n, src, dst, w, R, out), nprocs=2, join=True)
    got = np.load(out)
    P = ppr.transition_matrix(ppr.symmetric_weights(n, src, dst, w))[0]
    want = ppr.ppr_batch_power(P, R, 0.5)
    np.testing.assert_allclose(got, want, atol=1e-12)


def _stage_a_worker(rank, world, port, fe, Q, k, out_path):
    """Fact-sharded stage A, host logic (fact_stream.cu fact_stage_a with world > 1): every rank scores ITS fact rows
    [rank * ceil(F / world), ...), keeps its 8 best (score desc, row asc) and its (min, max); one all-gather of
    those per query; the merge of the `world` candidate lists is the global top-k and the global min / max."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    F = fe.shape[0]
    chunk = -(-F // world)
    lo, hi = min(F, rank * chunk), min(F, (rank + 1) * chunk)
    S = (Q @ fe[lo:hi].T).astype(np.float32)                       # [B, local rows]
    B = Q.shape[0]
    cand_score = np.full((B, 8), -np.inf, dtype=np.float32)
    cand_row = np.full((B, 8), -1, dtype=np.int64)
    mm = np.zeros((B, 2), dtype=np.float32)
    for b in range(B):
        if hi > lo:
            order = np.lexsort((np.arange(hi - lo), -S[b]))[:8]
            cand_score[b, :len(order)] = S[b, order]
            cand_row[b, :len(order)] = order + lo                  # local row -> global row (idx_offset)
            mm[b] = (S[b].min(), S[b].max())
        else:
            mm[b] = (np.inf, -np.inf)
    def gather(x):
        parts = [torch.zeros_like(torch.from_numpy(x)) for _ in range(world)]
        dist.all_gather(parts, torch.from_numpy(x))
        return np.stack([p.numpy() for p in parts])                # [world, B, ...]
    all_s, all_r, all_mm = gather(cand_score), gather(cand_row), gather(mm)
    top_idx = np.empty((B, k), dtype=np.int64)
    top_score = np.empty((B, k), dtype=np.float32)
    for b in range(B):
        s, r = all_s[:, b].ravel(), all_r[:, b].ravel()
        ok = r >= 0
        s, r = s[ok], r[ok]
        order = np.lexsort((r, -s))[:k]
        mn, mx = all_mm[:, b, 0].min(), all_mm[:, b, 1].max()
        top_idx[b] = r[order]
        top_score[b] = (s[order] - mn) / (mx - mn) if mx > mn else 1.0
    if rank == 0:
        np.savez(out_path, idx=top_idx, score=top_score)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("F", [37, 1000])
def test_two_rank_fact_sharded_stage_a_matches_the_oracle(tmp_path, F):
    from oracle import retrieve
    rng = np.random.default_rng(F)
    d = 16
    fe = rng.standard_normal((F, d)).astype(np.float32)
    fe /= np.linalg.norm(fe, axis=1, keepdims=True)
    fe[F // 2 + 1] = fe[3]                                         # an exact tie across the two shards
    Q = fe[rng.integers(0, F, 6)] + 0.3 * rng.standard_normal((6, d)).astype(np.float32)
    Q[0] = fe[3]
    out = str(tmp_path / "a.npz")
    mp.spawn(_stage_a_worker, args=(2, _free_port(), fe, Q, 5, out), nprocs=2, join=True)
    got = np.load(out)
    for b in range(6):
        fs32 = (fe @ Q[b]).astype(np.float32)
        want = np.lexsort((np.arange(F), -fs32))[:5]               # score desc, row asc: the library's tie policy
        assert list(got["idx"][b]) == list(want)
        np.testing.assert_allclose(got["score"][b], retrieve.min_max_normalize(fs32)[want], rtol=1e-6)


def test_balanced_row_bounds_split_work_not_rows():
    """The node-range partition handed to hrag_comm_set_row_bounds: contiguous, covering, equal shares of
    (non-zeros + 4 per row) -- on the synthetic KGs the passage rows are 3x denser than the entity rows."""
    from hipporag_b200 import balanced_row_bounds, synth
    from hipporag_b200.engine import build_transition_csr
    kg = synth.make_kg(20_000, 200_000, seed=1)
    row_ptr, _, _ = build_transition_csr(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    for world in (1, 2, 3, 8):
        b = balanced_row_bounds(row_ptr, world)
        assert b[0] == 0 and b[-1] == kg.n_nodes and np.all(np.diff(b) >= 0) and len(b) == world + 1
        cost = np.array([(row_ptr[b[i + 1]] - row_ptr[b[i]]) + 4 * (b[i + 1] - b[i]) for i in range(world)], dtype=float)
        assert cost.max() / cost.mean() < 1.01
    eq = np.array([row_ptr[min(kg.n_nodes, (i + 1) * 2500)] - row_ptr[i * 2500] for i in range(8)], dtype=float)
    assert eq.max() / eq.mean() > 1.8            # what the equal-row-count split would have cost the last rank
    # degenerate: more ranks than rows
    b = balanced_row_bounds(np.array([0, 3, 5]), 4)
    assert b[0] == 0 and b[-1] == 2 and np.all(np.diff(b) >= 0)


def _balanced_worker(rank, world, port, n, src, dst, w, R, out_path):
    """The sharded solve with the WORK-BALANCED partition (unequal row ranges): every rank sweeps rows
    [bounds[rank], bounds[rank + 1]) and the exchange is one broadcast per owner (comm.cu exchange_rows_bytes with
    row_bounds set; on devices the fused kernel writes the same ranges into the peers' buffers)."""
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hipporag_b200.engine import balanced_row_bounds, build_transition_csr, slice_csr_rows
    import scipy.sparse as sp
    row_ptr, col, val = build_transition_csr(n, src, dst, w)
    bounds = balanced_row_bounds(row_ptr, world)
    lo, hi = int(bounds[rank]), int(bounds[rank + 1])
    rp, c, v = slice_csr_rows(row_ptr, col, val, lo, hi)
    P_local = sp.csr_matrix((v.astype(np.float64), c, rp), shape=(hi - lo, n))
    X = torch.from_numpy(R.copy())
    V = R.copy()
    for _ in range(60):
        X[lo:hi] = torch.from_numpy(0.5 * (P_local @ X.numpy()) + V[lo:hi])
        for owner in range(world):                                       # grouped broadcasts, unequal counts
            a, b = int(bounds[owner]), int(bounds[owner + 1])
            if b > a:
                blk = X[a:b].contiguous()
                dist.broadcast(blk, src=owner)
                X[a:b] = blk
    if rank == 0:
        Z = X.numpy()
        np.save(out_path, Z / Z.sum(axis=0, keepdims=True))
    dist.barrier()
    dist.destroy_process_group()


def test_two_rank_work_balanced_partition_matches_oracle(tmp_path):
    rng = np.random.default_rng(5)
    n = 300
    # the last 30 vertices are "passages" with 4x the degree, as on the synthetic KGs: equal row counts would be unbalanced
    src = np.concatenate([rng.integers(0, 270, 900), rng.integers(270, 300, 1200)])
    dst = np.concatenate([rng.integers(0, 270, 900), rng.integers(0, 270, 1200)])
    keep = src != dst
    src, dst = src[keep], dst[keep]
    w = rng.random(src.shape[0]) + 0.2
    R = rng.random((n, 3)) * (rng.random((n, 3)) < 0.3)
    R[0] += 0.1
    from hipporag_b200.engine import balanced_row_bounds, build_transition_csr
    b = balanced_row_bounds(build_transition_csr(n, src, dst, w)[0], 2)
    assert b[1] > n // 2                                  # the dense tail makes the second range shorter
    out = str(tmp_path / "pi.npy")
    mp.spawn(_balanced_worker, args=(2, _free_port(), n, src, dst, w, R, out), nprocs=2, join=True)
    got = np.load(out)
    P = ppr.transition_matrix(ppr.symmetric_weights(n, src, dst, w))[0]
    np.testing.assert_allclose(got, ppr.ppr_batch_power(P, R, 0.5), atol=1e-6)     # fp32 CSR values (val is float32)
