"""Column-sharded cfg5 aggregation (SURVEY 8e "alternative to measure") -- EXPERIMENTAL, never run.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node R --master-addr 127.0.0.1 \
        --master-port 29511 scripts/bench_colshard.py [--steps 10]

Every rank builds the whole graph and owns 128/R feature columns.  Reports, max over ranks: the
aggregation alone (no communication), the all-to-all that re-shards [N, D/R] -> [N/R, D] for the dense
transform, and both together, next to the row-partition numbers of bench.py."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--edges", type=int, default=100_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl")
    import pgl_b200 as pgl
    import pgl_b200.nn.functional as GF
    from pgl_b200.distributed import ColumnShardedGraph
    edges = bench.gen_edges(torch, args.nodes, args.edges, 0.8, 20240922, dev)
    g = pgl.Graph(edges=edges, num_nodes=args.nodes)
    norm = GF.degree_norm(g)
    cs = ColumnShardedGraph(g, args.dim, world, rank)
    gen = torch.Generator(device=dev).manual_seed(1 + rank)
    x = torch.randn(args.nodes, cs.d_local, device=dev, generator=gen)
    ev = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731

    def timed(fn):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        a, b = ev(), ev()
        a.record()
        for _ in range(args.steps):
            fn()
        b.record()
        torch.cuda.synchronize()
        t = torch.tensor([a.elapsed_time(b) / args.steps], device=dev, dtype=torch.float64)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    t_agg = timed(lambda: cs.gcn_aggregate(x, norm))
    t_a2a = timed(lambda: cs.to_rows(x)) if world > 1 else 0.0
    t_both = timed(lambda: cs.to_rows(cs.gcn_aggregate(x, norm)))
    if rank == 0:
        d = cs.d_local
        b_alg = args.edges * (4 * d + 8) + args.nodes * 4 * d + (args.nodes + 1) * 8 + 2 * args.nodes * 4
        print(json.dumps({"workload": "cfg5, column-sharded %d ways (%d columns per GPU)" % (world, d),
                          "aggregate_ms": t_agg, "reshard_all_to_all_ms": t_a2a, "aggregate_plus_reshard_ms": t_both,
                          "edges_per_s_aggregate": args.edges / (t_agg * 1e-3),
                          "edges_per_s_with_reshard": args.edges / (t_both * 1e-3),
                          "per_gpu_alg_GBs": b_alg / t_agg / 1e6,
                          "per_gpu_roofline_frac": b_alg / t_agg / 1e6 / bench.peaks()[0]}))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
