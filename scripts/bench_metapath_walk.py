"""Times metapath walks (pgl.sampling.metapath_randomwalk, csrc/walk.cu) on the seeded MAG-like graph of
scripts/bench_hetero_sampler.py: 10^7 nodes (5M paper, 4.9M author, 0.1M institution), 10^8 edges in 5 relations.

Every paper node is a walker, walk length 40.  Calls, alternating call by call after --warmup rounds:
  - metapath rev_writes-writes (paper -> author -> paper) and cites-rev_writes-writes (length 3);
  - metapath [cites] (M = 1: the metapath kernel on one relation) and random_walk on graph["cites"], the same walks
    bit for bit (checked once here), so the two kernels' times compare directly.
Kernel time is CUDA events around the ops call (the [n, 40] output allocation included), median and p10 / p90 over
--reps rounds.  Reported per call: G steps/s (steps = nodes written after the start), the share of walks that end
early, and the byte model of DESIGN section 4.9 -- two dependent random 32-byte sectors per step (the indptr pair,
then the column) -- over kernel time, named as a model.  A host baseline restates the reference example's loop
(examples/metapath2vec/datasets/sampling.py metapath_randomwalk: per step one successor sample per live walker, a
Python list per node) in numpy on --host-walkers walkers, one thread; it is a reported baseline, not a target.  The
card's name, power limit and max SM clock are read in the same run.

    python scripts/bench_metapath_walk.py [--reps 7] [--warmup 2] [--json FILE]
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
from bench_hetero_sampler import mag_like  # noqa: E402
from pgl_b200 import ops  # noqa: E402

METAPATHS = {"rev_writes-writes": ["rev_writes", "writes"],
             "cites-rev_writes-writes": ["cites", "rev_writes", "writes"],
             "[cites]": ["cites"]}


def host_baseline(csrs, metapath, starts, walk_length, rng):
    """The reference example's loop in numpy: per step, the successors of every live walker's node as a Python list,
    one uniform pick each; a walker without successors stops.  Returns the steps taken."""
    walks = [[int(v)] for v in starts]
    ids, cur = np.arange(len(starts)), np.asarray(starts)
    for t in range(walk_length - 1):
        indptr, cols = csrs[metapath[t % len(metapath)]]
        succs = [cols[indptr[u]:indptr[u + 1]].tolist() for u in cur]
        mask = np.array([len(s) > 0 for s in succs], bool)
        if not mask.any():
            break
        ids, cur = ids[mask], cur[mask]
        nxt = [s[int(rng.integers(len(s)))] for s, m in zip(succs, mask) if m]
        for w, v in zip(ids, nxt):
            walks[w].append(v)
        cur = np.array(nxt, np.int64)
    return sum(len(w) - 1 for w in walks)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--papers", type=int, default=5_000_000)
    ap.add_argument("--authors", type=int, default=4_900_000)
    ap.add_argument("--institutions", type=int, default=100_000)
    ap.add_argument("--edges", type=int, default=100_000_000)
    ap.add_argument("--walk-length", type=int, default=40)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--host-walkers", type=int, default=2000)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_metapath_walk.py times GPU kernels and needs a CUDA device"
    torch.cuda.set_device(0)
    res = {"gpu": gpu_info(), "papers": args.papers, "authors": args.authors, "institutions": args.institutions,
           "edges": args.edges, "walk_length": args.walk_length, "reps": args.reps}
    print(json.dumps({"gpu": res["gpu"]}), flush=True)

    edges, n, types = mag_like(args.papers, args.authors, args.institutions, args.edges, seed=11)
    hg = pgl.HeterGraph(edges=edges, num_nodes=n, node_types=types)
    del edges
    L = args.walk_length
    nodes = torch.arange(args.papers, device="cuda")
    csr = {e: hg[e]._walk_csr()[:2] for e in ("cites", "writes", "rev_writes")}
    torch.cuda.synchronize()

    def metapath_call(mp):
        ip, cols = zip(*[csr[e] for e in METAPATHS[mp]])
        return lambda: ops.metapath_walk(ip, cols, n, nodes, L, 1234)

    calls = {mp: metapath_call(mp) for mp in METAPATHS}
    calls["random_walk cites"] = lambda: ops.random_walk(csr["cites"][0], csr["cites"][1], n, nodes, L, 1234)
    assert torch.equal(calls["[cites]"](), calls["random_walk cites"]()), "M = 1 is not random_walk"

    times = {k: [] for k in calls}
    counts = {}
    names = list(calls)
    for r in range(args.warmup + args.reps):
        for k in (names if r % 2 == 0 else names[::-1]):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = calls[k]()
            b.record()
            torch.cuda.synchronize()
            if r >= args.warmup:
                times[k].append(a.elapsed_time(b))
            if k not in counts:
                length = (out >= 0).sum(1)
                counts[k] = (int(length.sum().item()) - int(nodes.numel()), float((length < L).float().mean().item()))
            del out
    rows = []
    for k in names:
        med, p10, p90 = stats(times[k])
        steps, early = counts[k]
        row = {"call": k, "walkers": int(nodes.numel()), "walk_length": L, "kernel_ms_median": round(med, 3),
               "kernel_ms_p10": round(p10, 3), "kernel_ms_p90": round(p90, 3), "steps": steps,
               "G_steps_per_s": steps / (med / 1e3) / 1e9, "early_end_share": early,
               "byte_model_GBps": steps * 2 * 32 / (med / 1e3) / 1e9}
        rows.append(row)
        print(json.dumps(row), flush=True)
    res["calls"] = rows

    rng = np.random.default_rng(0)
    host = {e: tuple(t.cpu().numpy() for t in csr[e]) for e in csr}
    starts = rng.integers(0, args.papers, args.host_walkers)
    res["host_baseline"] = []
    for mp in ("rev_writes-writes", "cites-rev_writes-writes"):
        t0 = time.perf_counter()
        steps = host_baseline(host, METAPATHS[mp], starts, L, rng)
        dt = time.perf_counter() - t0
        row = {"host_baseline": mp, "walkers": args.host_walkers, "walk_length": L, "threads": 1,
               "seconds": round(dt, 3), "M_steps_per_s": steps / dt / 1e6}
        res["host_baseline"].append(row)
        print(json.dumps(row), flush=True)
    res["peak_gb"] = torch.cuda.max_memory_allocated() / 1e9
    print(json.dumps(res), flush=True)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
