"""Times skip-gram pair generation and alias negative sampling (csrc/skipgram.cu) from device walks.

    python scripts/bench_skipgram.py [--reps 5] [--host-walks 512] [--out FILE]

Workloads, all on an RMAT (0.57, 0.19, 0.19, 0.05) graph of 2^20 nodes and 10^7 edges (many sinks):
  - deepwalk: 512 walks of 40 nodes, window 10, 20 negatives per pair (the reference's examples/deepwalk/config.yaml);
  - metapath2vec: 512 metapath walks of 24 nodes over a two-relation split of the graph, window 3, 5 negatives
    (examples/metapath2vec/config.yaml);
  - all_nodes: every node walks 80 steps (81 nodes), window 10, 1 negative per pair.
Negatives come from the alias table of outdegree^0.75.  Reported per workload:
  - kernel times (torch.profiler, CUDA activity, in a run of its own) of the count, the scan (its three launches),
    the fill and the sample, the median over --reps;
  - pairs per second over count + scan + fill;
  - bytes written (16 per pair, 8 per negative) over fill and over sample time, against 3.35 TB/s (H100 SXM HBM3);
  - the batch time from walk to negatives (CUDA events, profiler off), and the reference-style host pipeline on the
    same walks -- walks copied to the host, graph_kernel.skip_gram_gen_pair once per walk in a Python loop, negatives
    by np.random -- timed on the first --host-walks walks and scaled to the batch;
  - the card's name and power limit, read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (graph generators)
import pgl_b200 as pgl  # noqa: E402
from pgl_b200 import graph_kernel as gk  # noqa: E402

HBM = 3.35e12
KERNELS = {"count": ("skipgram_count_kernel",), "scan": ("scan_tile_sums_kernel", "scan_sums_kernel",
                                                         "scan_apply_kernel"),
           "fill": ("skipgram_fill_kernel",), "sample": ("alias_sample_kernel",)}


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "not read"}


def workloads(g, hg, n):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    starts = torch.randint(0, n, (512,), generator=gen, device="cuda")
    return [
        ("deepwalk", lambda s: pgl.sampling.random_walk(g, starts, 40, seed=s), 10, 20),
        ("metapath2vec", lambda s: pgl.sampling.metapath_randomwalk(hg, starts, "r0-r1", 24, seed=s), 3, 5),
        ("all_nodes", lambda s: pgl.sampling.random_walk(g, torch.arange(n, device="cuda"), 81, seed=s), 10, 1),
    ]


def batch(walk, win, neg, alias, events, s):
    walks = walk(s)
    src, pos = pgl.sampling.skip_gram_pairs(walks, win, seed=s)
    negs = pgl.sampling.alias_sample(alias, events, (src.numel(), neg), seed=s)
    return walks, src, pos, negs


def kernel_times(fn, reps):
    from torch.profiler import ProfilerActivity, profile
    per = {k: [] for k in KERNELS}
    for _ in range(reps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        tot = {k: 0.0 for k in KERNELS}
        for ev in prof.events():
            for k, names in KERNELS.items():
                if any(nm in ev.name for nm in names):
                    tot[k] += ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        for k in KERNELS:
            per[k].append(tot[k] * 1e-6)   # us -> s
    return {k: float(np.median(v)) for k, v in per.items()}


def host_pipeline(walks, win, neg, n, count):
    rows = walks[:count].cpu().numpy()
    t0 = time.perf_counter()
    s = []
    for row in rows:
        a, _ = gk.skip_gram_gen_pair(row[row >= 0], win)
        s += a
    np.random.randint(0, n, (len(s), neg))
    return (time.perf_counter() - t0) / len(rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--host-walks", type=int, default=512)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_skipgram.py needs a CUDA device"
    torch.cuda.set_device(0)
    n = 1 << 20
    edges = bench.rmat_edges(torch, 20, 10_000_000, seed=1, device="cuda")
    g = pgl.Graph(edges=edges, num_nodes=n)
    half = edges.shape[0] // 2
    hg = pgl.HeterGraph(edges={"r0": edges[:half].cpu().numpy(), "r1": edges[half:].cpu().numpy()}, num_nodes=n,
                        node_types=np.zeros(n, np.int64)).tensor()
    alias, events = pgl.sampling.alias_table(g.outdegree().double() ** 0.75)
    res = {"card": card(), "graph": {"nodes": n, "edges": int(edges.shape[0])}, "workloads": []}
    for name, walk, win, neg in workloads(g, hg, n):
        for s in range(2):   # warm-up
            out = batch(walk, win, neg, alias, events, s)
        del out
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for s in range(a.reps):
            t0.record()
            walks, src, pos, negs = batch(walk, win, neg, alias, events, 10 + s)
            t1.record()
            torch.cuda.synchronize()
            times.append(t0.elapsed_time(t1) * 1e-3)
            pairs, B = src.numel(), walks.shape[0]
            del src, pos, negs
        kt = kernel_times(lambda: batch(walk, win, neg, alias, events, 10), a.reps)
        host_per_walk = host_pipeline(walks, win, neg, n, min(a.host_walks, B))
        sg = kt["count"] + kt["scan"] + kt["fill"]
        row = {"workload": name, "walks": B, "walk_len": int(walks.shape[1]), "win_size": win, "negatives": neg,
               "pairs": pairs, "kernel_s": kt, "pairs_per_s": pairs / sg if sg else None,
               "fill_write_TBps": 16 * pairs / kt["fill"] / 1e12 if kt["fill"] else None,
               "fill_share_of_hbm": 16 * pairs / kt["fill"] / HBM if kt["fill"] else None,
               "sample_write_TBps": 8 * pairs * neg / kt["sample"] / 1e12 if kt["sample"] else None,
               "sample_share_of_hbm": 8 * pairs * neg / kt["sample"] / HBM if kt["sample"] else None,
               "batch_s_median": float(np.median(times)),
               "host_pipeline_s_per_walk": host_per_walk, "host_walks_timed": min(a.host_walks, B),
               "host_pipeline_s_scaled": host_per_walk * B}
        res["workloads"].append(row)
        print(json.dumps(row), flush=True)
        del walks
        torch.cuda.empty_cache()
    print(json.dumps({"card": res["card"]}))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
