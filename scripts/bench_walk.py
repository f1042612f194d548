"""Times the random-walk kernels (csrc/walk.cu) with every node as a walker.

    python scripts/bench_walk.py [--graphs cfg5,rmat1m,rmat10m] [--depths 40,80] [--reps 3] [--out FILE]

Graphs: bench.py's cfg5 power-law graph (10M nodes / 100M edges, Chung-Lu exponent 0.8) and RMAT (0.57, 0.19, 0.19,
0.05) with 2^20 nodes / 10M edges and 10M nodes / about 100M edges (scale 24, edges with an id >= 10^7 dropped).
Rules: random_walk, then node2vec_walk at (p, q) = (0.25, 4) and (4, 0.25).  Reported per run:
  - walk steps per second (steps = nodes written after the start, over the median kernel call of --reps);
  - rejection trials per step and the share of steps that took the exact fallback (node2vec);
  - a byte model, named as such: dependent random 32-byte sectors per step (random_walk: the indptr pair and the
    column, 2; node2vec: 2 plus, per trial, the column and the indptr pair of prev plus one sector per binary-search
    probe, log2(mean degree) + 1), times 32 bytes, over kernel time;
  - a host baseline: a restatement of the reference's pgl/sampling/walk.py loop (numpy, one Python call per walker per
    node2vec step) timed on a stated subset of walkers on one core.  It is a reported baseline, not a target.
The card's name and power limit are read in the same run."""
import argparse
import json
import math
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
from pgl_b200 import ops  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "not read"}


def make_graph(name, dev):
    if name == "cfg5":
        n = 10_000_000
        edges = bench.gen_edges(torch, n, 100_000_000, 0.8, 20240922, dev)
    elif name == "rmat1m":
        n = 1 << 20
        edges = bench.rmat_edges(torch, 20, 10_000_000, seed=1, device=dev)
    else:
        n = 10_000_000
        edges = bench.rmat_edges(torch, 24, 100_000_000, seed=1, device=dev)
        edges = edges[(edges[:, 0] < n) & (edges[:, 1] < n)].contiguous()
    return pgl.Graph(edges=edges, num_nodes=n), n, int(edges.shape[0])


def host_baseline(indptr, cols, nodes, depth, p, q, rng, budget_s):
    """The reference's walk loop restated in numpy (pgl/sampling/walk.py:23-122 with graph_kernel.node2vec_sample's
    per-walker weight loop in Python): returns (steps taken, walkers finished).  node2vec stops after the walker that
    crosses budget_s seconds (a hub row of 10^6 successors is a Python loop per step)."""
    t0 = time.perf_counter()
    succ = lambda u: cols[indptr[u]:indptr[u + 1]]  # noqa: E731
    walks = [[int(v)] for v in nodes]
    if p == 1.0 and q == 1.0:
        cur_ids, cur = np.arange(len(nodes)), np.array(nodes)
        for _ in range(depth - 1):
            succs = [succ(u) for u in cur]
            mask = np.array([len(s) > 0 for s in succs])
            if not mask.any():
                break
            cur_ids, cur = cur_ids[mask], cur[mask]
            succs = [s for s, m in zip(succs, mask) if m]
            idx = np.floor(rng.random(len(succs)) * [len(s) for s in succs]).astype(np.int64)
            nxt = [int(s[i]) for s, i in zip(succs, idx)]
            for w, v in zip(cur_ids, nxt):
                walks[w].append(v)
            cur = np.array(nxt)
    else:
        for w in range(len(nodes)):
            if time.perf_counter() - t0 > budget_s:
                walks = walks[:w]
                break
            c, pr, pset = walks[w][0], -1, set()
            for _ in range(depth):
                s = succ(c)
                if len(s) == 0:
                    break
                wt = [1.0 / p if v == pr else (1.0 if v in pset else 1.0 / q) for v in s.tolist()]
                x = rng.random() * sum(wt)
                for v, t in zip(s.tolist(), wt):
                    x -= t
                    if x <= 0:
                        break
                walks[w].append(v)
                pr, pset, c = c, set(s.tolist()), v
    return sum(len(w) - 1 for w in walks), len(walks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--graphs", default="cfg5,rmat1m,rmat10m")
    ap.add_argument("--depths", default="40,80")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--host-walkers", type=int, default=2000)
    ap.add_argument("--host-budget-s", type=float, default=60.0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_walk.py times the GPU kernels and needs a CUDA device"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = {"card": card(), "host_cores": os.cpu_count()}
    print(json.dumps(info), flush=True)
    results = [info]
    rules = [("random_walk", 1.0, 1.0), ("node2vec_walk", 0.25, 4.0), ("node2vec_walk", 4.0, 0.25)]
    for gname in args.graphs.split(","):
        g, n, e = make_graph(gname, dev)
        t0 = time.perf_counter()
        indptr, cols, srt = g._walk_csr(row_sorted=True)
        torch.cuda.synchronize()
        t_sorted = time.perf_counter() - t0
        deg_mean = e / n
        nodes = torch.arange(n, device=dev)
        for depth in (int(d) for d in args.depths.split(",")):
            for rule, p, q in rules:
                stats = torch.zeros(2, dtype=torch.int64, device=dev)

                def call():
                    if rule == "random_walk":
                        return ops.random_walk(indptr, cols, n, nodes, depth, 1234)
                    return ops.node2vec_walk(indptr, cols, srt, n, nodes, depth, p, q, False, 1234, stats)
                out = call()  # warm-up
                del out
                times = []
                for _ in range(args.reps):
                    stats.zero_()
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    out = call()
                    b.record()
                    torch.cuda.synchronize()
                    times.append(a.elapsed_time(b) / 1e3)
                    steps = int((out >= 0).sum().item()) - n
                    del out
                t = float(np.median(times))
                trials, fallbacks = (int(x) for x in stats.tolist())
                if rule == "random_walk":
                    trials, sectors = steps, 2.0
                else:
                    sectors = 2.0 + trials / steps * (3.0 + math.log2(max(deg_mean, 1.0)))
                r = {"graph": gname, "nodes": n, "edges": e, "depth": depth, "rule": rule, "p": p, "q": q,
                     "kernel_s_median": round(t, 4), "kernel_s_all": [round(x, 4) for x in times],
                     "steps": steps, "steps_per_s": steps / t, "trials_per_step": trials / steps,
                     "fallback_share": fallbacks / steps if rule != "random_walk" else 0.0,
                     "byte_model_sectors_per_step": round(sectors, 2),
                     "byte_model_GBps": steps * sectors * 32 / t / 1e9,
                     "row_sorted_copy_build_s": round(t_sorted, 3)}
                print(json.dumps(r), flush=True)
                results.append(r)
        # host baseline on a subset of walkers, depth 40
        hp, hc = indptr.cpu().numpy(), cols.cpu().numpy()
        rng = np.random.default_rng(0)
        sub = rng.integers(0, n, args.host_walkers)
        for rule, p, q in rules:
            t0 = time.perf_counter()
            steps, done = host_baseline(hp, hc, sub, 40, p, q, rng, args.host_budget_s)
            dt = time.perf_counter() - t0
            r = {"graph": gname, "host_baseline": rule, "p": p, "q": q, "walkers": done, "depth": 40,
                 "threads": 1, "seconds": round(dt, 3), "steps_per_s": steps / dt}
            print(json.dumps(r), flush=True)
            results.append(r)
        del g, indptr, cols, srt, nodes
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
