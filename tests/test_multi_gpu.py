"""Node-range-sharded PPR on 2+ GPUs (one process per GPU, NCCL all-gather per sweep) against the
oracle.  Needs >= 2 visible GPUs; skipped otherwise."""
import os
import socket

import numpy as np
import pytest

from oracle import ppr

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_path, fused=False):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)      # only carries the NCCL id
    from hipporag_b200 import Engine, synth
    kg = synth.make_kg(30_000, 300_000, seed=2)
    rng = np.random.default_rng(0)
    R = np.zeros((21, kg.n_nodes), np.float32)
    R[:, kg.passage_vid] = 0.05 * rng.random((21, kg.n_pass), dtype=np.float32)
    for b in range(21):
        R[b, rng.integers(0, kg.n_ent, 5)] = rng.random(5, dtype=np.float32)
    ids = [Engine.new_comm_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    e = Engine(rank, shard_mode=1)
    e.init_comm(ids[0], rank, world)
    e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    if fused:                                   # K5: peer stores over NVLink instead of the NCCL all-gather
        handles = [None] * world
        dist.all_gather_object(handles, e.p2p_export())
        e.p2p_import(handles)
    got = e.ppr(R)
    got2 = e.ppr(R[:18])                        # a second call: epochs keep counting across calls (18 > 16: same solver)
    assert np.array_equal(got2, got[:18])
    got3 = e.ppr(R[:5])                         # <= 16 columns: the fp32 solver, NCCL all-gather exchange
    assert np.max(np.abs(got3 - got[:5]) / got[:5].max(axis=1, keepdims=True)) < 2e-5
    if rank == 0:
        np.save(out_path, got)
    st = e.stats()
    assert st["ms_comm"] > 0
    dist.barrier()
    e.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("fused", [False, True])
def test_sharded_ppr_two_gpus(tmp_path, fused):
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from hipporag_b200 import synth
    out = str(tmp_path / "pi.npy")
    mp.spawn(_worker, args=(2, _free_port(), out, fused), nprocs=2, join=True)
    got = np.load(out)
    kg = synth.make_kg(30_000, 300_000, seed=2)
    rng = np.random.default_rng(0)
    R = np.zeros((21, kg.n_nodes), np.float32)
    R[:, kg.passage_vid] = 0.05 * rng.random((21, kg.n_pass), dtype=np.float32)
    for b in range(21):
        R[b, rng.integers(0, kg.n_ent, 5)] = rng.random(5, dtype=np.float32)
    P = ppr.transition_matrix(ppr.symmetric_weights(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w))[0]
    want = ppr.ppr_batch_power(P, R.T.astype(np.float64), 0.5).T
    assert np.max(np.abs(got - want) / want.max(axis=1, keepdims=True)) < 2e-5


def _retrieve_worker(rank, world, port, out_path, fused):
    import torch
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from hipporag_b200 import Engine, synth
    kg = synth.make_kg(20_000, 200_000, seed=4)
    d = 64
    fe, pe = synth.unit_rows(kg.n_facts, d, 1), synth.unit_rows(kg.n_pass, d, 2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 100, seed=3)          # 4 sub-batches of 32 (ragged tail)
    ids = [Engine.new_comm_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    e = Engine(rank, shard_mode=1)
    e.init_comm(ids[0], rank, world)
    e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    if fused:
        handles = [None] * world
        dist.all_gather_object(handles, e.p2p_export())
        e.p2p_import(handles)
    e.load_tables(kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    e.load_embeddings(fe, pe)
    for _ in range(2):                                                # twice: epochs continue across calls
        idx, score, nv = e.stage_a(qf, 5)
        out_ids, out_scores = e.stage_b(qp, idx, score, topk=50)
    if rank == 0:
        np.savez(out_path, ids=out_ids, scores=out_scores)
    dist.barrier()
    e.close()
    dist.destroy_process_group()


@pytest.mark.parametrize("fused", [False, True])
def test_sharded_retrieve_two_gpus(tmp_path, fused):
    """Whole stage A/B path with the graph node-range-sharded over 2 GPUs (NCCL all-gather or K5)."""
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    from hipporag_b200 import synth
    from oracle import retrieve
    from tests.util import assert_topk_matches
    out = str(tmp_path / "out.npz")
    mp.spawn(_retrieve_worker, args=(2, _free_port(), out, fused), nprocs=2, join=True)
    got = np.load(out)
    kg = synth.make_kg(20_000, 200_000, seed=4)
    d = 64
    fe, pe = synth.unit_rows(kg.n_facts, d, 1), synth.unit_rows(kg.n_pass, d, 2)
    qf, qp, _ = synth.make_queries(kg, fe, pe, 100, seed=3)
    P = ppr.transition_matrix(ppr.symmetric_weights(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w))[0]
    tb = retrieve.Tables(kg.n_nodes, kg.passage_vid, kg.fact_subj_vid, kg.fact_obj_vid, kg.ent_chunk_count)
    for q in (0, 31, 32, 64, 99):
        o = retrieve.retrieve_one(P, tb, fe, pe, qf[q], qp[q], top_k=None)
        full = np.empty(len(o["ids"]))
        full[o["ids"]] = o["scores"]
        assert_topk_matches(got["ids"][q], got["scores"][q], full, 50, what=f"sharded query {q}")
