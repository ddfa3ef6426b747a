#!/usr/bin/env python
"""Node-range-sharded mixed-precision sweep: NCCL all-gather per sweep vs K5 fused peer stores.
    torchrun --nproc-per-node G tools/sharded_sweep_bench.py [C3]
"""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
from bench import WORKLOADS

def main():
    name = sys.argv[1] if len(sys.argv) > 1 else "C3"
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("gloo")
    from hipporag_b200 import Engine, synth
    w = WORKLOADS[name]
    kg = synth.make_kg(w["n_nodes"], w["n_edges"], seed=0)
    ids = [Engine.new_comm_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    e = Engine(int(os.environ["LOCAL_RANK"]), shard_mode=1)
    e.init_comm(ids[0], rank, world)
    e.load_graph(kg.n_nodes, kg.edge_src, kg.edge_dst, kg.edge_w)
    dist.barrier()
    ms_nccl = e.bench_sweep(32, 30, 2)
    dist.barrier()
    handles = [None] * world
    dist.all_gather_object(handles, e.p2p_export())
    e.p2p_import(handles)
    dist.barrier()
    ms_p2p = e.bench_sweep(32, 30, 2)
    t = torch.tensor([ms_nccl, ms_p2p], dtype=torch.float64)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    if rank == 0:
        print(json.dumps({"workload": name, "gpus": world, "ms_per_sweep_nccl_allgather": round(float(t[0]), 4),
                          "ms_per_sweep_fused_peer_stores": round(float(t[1]), 4)}), flush=True)
    dist.barrier()
    e.close()
    dist.destroy_process_group()

if __name__ == "__main__":
    main()
