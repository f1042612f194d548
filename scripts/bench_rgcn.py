"""RGCNConv on a tensor-mode HeterGraph (the fused relation-typed aggregation, ops.rgcn_aggregate) against the same
layer on the equivalent dict of Graphs (the reference's per-relation loop: R matmuls, R send_recv(mean), R adds),
alternating inside every round.

Two workloads:
  * example: shaped like the reference's R-GCN example (examples/rgcn) -- N = 2^15 nodes, R = 64 relations with
    Zipf-distributed sizes, about 2e5 edges, RGCNConv(64 -> 64, num_bases = 8); many relations, few edges each;
  * rmat: cfg3's graph (RMAT scale 20, 10M edges, bench_gat.rmat) with the edges split uniformly into R = 8
    relations, RGCNConv(128 -> 128) without bases; few relations, many edges each.
For each: inference forward and training forward + backward (median, p10, p90 over all rounds), the peak memory of
one training step, and the library launches of each.  The outputs of both routes are compared at full size first.

    python scripts/bench_rgcn.py [--rounds 5] [--steps 10] [--json FILE]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
import pgl_b200 as pgl  # noqa: E402
from bench_gat import rmat  # noqa: E402
from bench_half import gpu_info, stats  # noqa: E402


def example_edges(n, R, e, seed=7):
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, R + 1)
    sizes = np.maximum(1, np.round(e * p / p.sum())).astype(np.int64)
    return [torch.as_tensor(np.stack([rng.integers(0, n, s), rng.integers(0, n, s)], 1)).cuda() for s in sizes]


def rmat_edges(R, seed=3):
    e = rmat(20, 10_000_000)
    rel = torch.randint(0, R, (e.shape[0],), generator=torch.Generator(device="cuda").manual_seed(seed), device="cuda")
    return [e[rel == r].contiguous() for r in range(R)], 1 << 20


def timed(fn, steps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return out


def peak_gb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 1e9


def launches(fn):
    torch.cuda.synchronize()
    l0 = pgl.ops.launch_count()
    fn()
    torch.cuda.synchronize()
    return pgl.ops.launch_count() - l0


def run(name, edge_lists, n, d, num_bases, rounds, steps):
    R = len(edge_lists)
    etypes = ["r%d" % i for i in range(R)]
    hg = pgl.HeterGraph(edges=dict(zip(etypes, edge_lists)), num_nodes=n, node_types=np.zeros(n, np.int64))
    graphs = {t: hg[t] for t in etypes}
    torch.manual_seed(0)
    conv = pgl.nn.RGCNConv(d, d, etypes, num_bases=num_bases).cuda()
    x = torch.randn((n, d), device="cuda", requires_grad=True)
    gout = torch.randn((n, d), device="cuda")
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    hg.typed_csr(etypes, x.device)
    t1.record()
    torch.cuda.synchronize()
    build_ms = t0.elapsed_time(t1)
    with torch.no_grad():
        a, b = conv(hg, x), conv(graphs, x)
    err = float((a - b).abs().max() / b.abs().max())
    assert err <= 1e-4, err
    routes = {"fused": hg, "old": graphs}

    def fwd(g):
        with torch.no_grad():
            conv(g, x)

    def train(g):
        conv(g, x).backward(gout)

    fwd_csr = hg.typed_csr(etypes, x.device)[0]
    res = {"workload": name, "nodes": n, "edges": int(sum(int(e.shape[0]) for e in edge_lists)), "relations": R,
           "dim": d, "num_bases": num_bases, "typed_csr_build_ms": build_ms, "max_rel_err_vs_old": err,
           # ops.rgcn_fused_pays: the layer's "fused" route is the per-relation one where this is False
           "fused_route_taken": pgl.ops.rgcn_fused_pays(fwd_csr, d, d),
           "staged_w_over_dense_rows": fwd_csr["tile_rels"] * d * d / (R * n * 2 * d)}
    # the forward kernel alone, whichever route the layer takes
    w3 = conv.weight.detach() if num_bases == 0 else torch.einsum("rb,bio->rio", conv.w_comp, conv.weight).detach()
    xd = x.detach()
    kern = timed(lambda: pgl.ops._rgcn_agg_raw(fwd_csr, xd, w3), steps * rounds)
    res["fwd_kernel_ms"] = dict(zip(("median", "p10", "p90"), stats(kern)))
    t = {(k, r): [] for k in ("fwd", "train") for r in routes}
    for _ in range(rounds):
        for r, g in routes.items():
            t[("fwd", r)] += timed(lambda: fwd(g), steps)
            t[("train", r)] += timed(lambda: train(g), steps)
    for (k, r), v in t.items():
        med, p10, p90 = stats(v)
        res["%s_%s_ms" % (k, r)] = {"median": med, "p10": p10, "p90": p90}
    for r, g in routes.items():
        res["train_peak_gb_%s" % r] = peak_gb(lambda: train(g))
        res["launches_fwd_%s" % r] = launches(lambda: fwd(g))
        res["launches_train_%s" % r] = launches(lambda: train(g))
    # per-round wins: is fused faster in every round?
    per = steps
    for k in ("fwd", "train"):
        f, o = t[(k, "fused")], t[(k, "old")]
        res["%s_fused_faster_every_round" % k] = all(
            np.median(f[i * per:(i + 1) * per]) < np.median(o[i * per:(i + 1) * per]) for i in range(rounds))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    info = {"gpu": gpu_info()}
    print(json.dumps(info), flush=True)
    out = [info]
    r = run("example", example_edges(1 << 15, 64, 200_000), 1 << 15, 64, 8, args.rounds, args.steps)
    print(json.dumps(r), flush=True)
    out.append(r)
    el, n = rmat_edges(8)
    r = run("rmat", el, n, 128, 0, args.rounds, args.steps)
    print(json.dumps(r), flush=True)
    out.append(r)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
