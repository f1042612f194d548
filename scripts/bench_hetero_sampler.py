"""HeteroNeighborSampler and mini-batch RGCNConv on a seeded synthetic graph with a MAG240M-like schema.

Graph: node types paper / author / institution (5M / 4.9M / 0.1M by default, 10^7 nodes), R = 5 relations
cites (paper -> paper), writes (author -> paper), rev_writes (paper -> author), affiliated (author -> institution),
rev_affiliated (institution -> author), 10^8 edges (50 / 20 / 20 / 5 / 5 %).  Sources are uniform inside their type,
destinations skewed (id = floor(n_type u^2)), so in-degrees follow a heavy tail.  Batches of 1024 distinct paper
targets, fan-outs [25, 15] on every relation, D = 128, two RGCNConv(128 -> 128) layers.

Per batch (median, p10, p90 over --batches after --warmup), in the same run:
  1. sampling: typed sampling + one reindex per layer (HeteroNeighborSampler's device work) against what a user does
     without it: per layer R sample_neighbors calls on the per-relation dst-CSRs, concatenation, a stable sort to
     node-major order, one reindex_graph.  The two alternate batch by batch.  Both end in a host read, so a host clock
     around each call measures the work.
  2. block construction: the whole sample_neighbors call of the sampler; of it, the device-to-host copy of the blocks'
     node ids with the node-type lookup; and, outside it, typed_csr on the two blocks (built when the layer first runs).
  3. training step on fresh blocks: x[nodes] gather, two RGCNConv layers forward + backward, the fused route (typed_csr
     of the blocks + ops.rgcn_aggregate) against the per-relation route (the blocks' Graphs), alternating.

    python scripts/bench_hetero_sampler.py [--batches 30] [--warmup 5] [--json FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import pgl_b200 as pgl  # noqa: E402
from bench_half import gpu_info, stats  # noqa: E402
from pgl_b200.sampling import reindex_graph, sample_neighbors, sample_typed_neighbors  # noqa: E402

ETYPES = ["cites", "writes", "rev_writes", "affiliated", "rev_affiliated"]


def mag_like(n_paper, n_author, n_inst, edges, seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    base = {"paper": 0, "author": n_paper, "inst": n_paper + n_author}
    size = {"paper": n_paper, "author": n_author, "inst": n_inst}
    plan = [("cites", "paper", "paper", 0.5), ("writes", "author", "paper", 0.2), ("rev_writes", "paper", "author", 0.2),
            ("affiliated", "author", "inst", 0.05), ("rev_affiliated", "inst", "author", 0.05)]
    out = {}
    for name, s, d, frac in plan:
        m = int(edges * frac)
        src = torch.randint(0, size[s], (m,), generator=gen, device="cuda") + base[s]
        u = torch.rand((m,), generator=gen, device="cuda")
        dst = (u * u * size[d]).long().clamp_(max=size[d] - 1) + base[d]
        out[name] = torch.stack([src, dst], 1)
        del src, dst, u
    n = n_paper + n_author + n_inst
    types = np.zeros(n, np.int8)
    types[n_paper:n_paper + n_author] = 1
    types[n_paper + n_author:] = 2
    return out, n, types


def typed_layers(csr, nodes, fanouts, num_nodes, seed):
    """HeteroNeighborSampler's device work per batch: per layer one typed sampling + one reindex."""
    for i, k in enumerate(fanouts):
        nb, rel, cnt = sample_typed_neighbors(csr["indptr"], csr["cols"], csr["rel"], nodes, [k] * len(ETYPES),
                                              seed=seed + i)
        _, _, nodes = reindex_graph(nodes, nb, cnt, num_nodes=num_nodes)
    return nodes


def per_relation_layers(csrs, nodes, fanouts, num_nodes, seed):
    """Without the typed sampler: R sample_neighbors calls per layer, concatenation, node-major order, one reindex."""
    for i, k in enumerate(fanouts):
        nbs, owners, cnt = [], [], None
        pos = torch.arange(int(nodes.shape[0]), device=nodes.device)
        for row, colptr in csrs:
            nb, c = sample_neighbors(row, colptr, nodes, sample_size=k, seed=seed + i)
            nbs.append(nb)
            owners.append(torch.repeat_interleave(pos, c))
            cnt = c if cnt is None else cnt + c
        nb = torch.cat(nbs)
        order = torch.sort(torch.cat(owners), stable=True).indices
        _, _, nodes = reindex_graph(nodes, nb.index_select(0, order), cnt, num_nodes=num_nodes)
    return nodes


def host_timed(fn):
    torch.cuda.synchronize()
    t = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t) * 1e3


def summary(v):
    med, p10, p90 = stats(v)
    return {"median": med, "p10": p10, "p90": p90}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--papers", type=int, default=5_000_000)
    ap.add_argument("--authors", type=int, default=4_900_000)
    ap.add_argument("--institutions", type=int, default=100_000)
    ap.add_argument("--edges", type=int, default=100_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--batches", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    fanouts = [25, 15]
    res = {"gpu": gpu_info(), "papers": args.papers, "authors": args.authors, "institutions": args.institutions,
           "edges": args.edges, "batch": args.batch, "fanouts": fanouts, "dim": args.dim}
    print(json.dumps({"gpu": res["gpu"]}), flush=True)

    edges, n, types = mag_like(args.papers, args.authors, args.institutions, args.edges, seed=11)
    hg = pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types)
    del edges
    sampler, init_ms = host_timed(lambda: pgl.sampling.HeteroNeighborSampler(hg, fanouts, seed=1))
    res["sampler_init_ms"] = init_ms
    csrs = [(hg[e].adj_dst_index._sorted_v, hg[e].adj_dst_index._indptr) for e in ETYPES]
    torch.cuda.synchronize()

    rng = np.random.default_rng(5)
    total = args.warmup + args.batches
    seeds = [torch.as_tensor(rng.choice(args.papers, args.batch, replace=False)).cuda() for _ in range(total)]

    t = {k: [] for k in ("typed", "per_relation", "sampler_total", "d2h_types", "block_typed_csr", "step_fused",
                         "step_per_relation")}
    torch.manual_seed(0)
    convs = [pgl.nn.RGCNConv(args.dim, args.dim, ETYPES).cuda() for _ in range(2)]
    x = torch.randn((n, args.dim), device="cuda")
    input_nodes = {"typed": [], "per_relation": []}
    for b, s in enumerate(seeds):
        keep = b >= args.warmup
        order = (("typed", lambda: typed_layers(sampler.csr, s, fanouts, n, 100 + b)),
                 ("per_relation", lambda: per_relation_layers(csrs, s, fanouts, n, 100 + b)))
        for name, fn in (order if b % 2 == 0 else order[::-1]):
            nodes, ms = host_timed(fn)
            if keep:
                t[name].append(ms)
                input_nodes[name].append(int(nodes.shape[0]))
        (blocks, nodes), ms = host_timed(lambda: sampler.sample_neighbors(s))
        # a block's nodes are the first num_nodes of the outermost layer's (reindex keeps earlier nodes first)
        _, ms_d2h = host_timed(lambda: [types[nodes[:int(blk.num_nodes)].cpu().numpy()] for blk, _ in blocks])
        _, ms_csr = host_timed(lambda: [blk.typed_csr(ETYPES, x.device) for blk, _ in blocks])
        if keep:
            t["sampler_total"].append(ms)
            t["d2h_types"].append(ms_d2h)
            t["block_typed_csr"].append(ms_csr)

        def step(route):
            h = x[nodes]
            for conv, (blk, nt) in zip(convs, blocks):
                g = blk if route == "fused" else {e: blk[e] for e in ETYPES}
                h = conv(g, h)[:nt]
            h.sum().backward()

        # fresh blocks for the timed steps: the fused route pays typed_csr, the other its per-relation indices
        (blocks, nodes) = sampler.sample_neighbors(s)
        names = ("fused", "per_relation") if b % 2 == 0 else ("per_relation", "fused")
        for route in names:
            _, ms = host_timed(lambda: step(route))
            if keep:
                t["step_" + route].append(ms)
        for conv in convs:
            conv.zero_grad(set_to_none=True)

    for k, v in t.items():
        res[k + "_ms"] = summary(v)
    res["input_nodes_median"] = {k: float(np.median(v)) for k, v in input_nodes.items()}
    res["sampling_speedup_median"] = res["per_relation_ms"]["median"] / res["typed_ms"]["median"]
    res["step_speedup_median"] = res["step_per_relation_ms"]["median"] / res["step_fused_ms"]["median"]
    res["peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    print(json.dumps(res), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
