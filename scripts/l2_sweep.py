"""How much L2 should the wide-row aggregation's hot set get, and what does streaming the per-slot source norms save?

Builds bench.py's cfg5 graph once (its own generators: Chung-Lu exponent 0.8, 10M nodes / 100M edges, 128-d f32) and
times ops._spmm_raw -- the GCN aggregation with both norm scalings, exactly bench.py's step -- for every hot-set budget
(packed ids made by ops.pack_cols(..., budget_bytes=)) x {source norm gathered per edge, streamed per slot}.  The
variants alternate inside every round, so drift of the shared machine spreads over all of them.  Every variant's
output is compared bit for bit with the first one's.

    python scripts/l2_sweep.py [--rounds 5] [--steps 10] [--budgets-mb 0,8,16,24,32,40,48,64] [--json FILE]

The model columns restate the byte model of the hot set: w_i = (i+1)^-0.8 over N sources, the k = budget / 512
heaviest rows are assumed to stay in L2 and every other row gather (512 B) to reach DRAM, plus output, packed ids,
indptr and the source norms (a 32-byte sector per slot with a cold source when gathered, 4 B per slot when streamed).
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import pgl_b200 as pgl  # noqa: E402
from pgl_b200 import ops  # noqa: E402

ROW = 512  # bytes of one 128-float feature row


def gpu_info():
    """Name, power limit and max SM clock: a read-only nvidia-smi query."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi failed"
    except (OSError, subprocess.TimeoutExpired) as ex:
        return "nvidia-smi unavailable: %r" % (ex,)


def model_gb(n, e, d, exponent, budget, streamed):
    """Modelled DRAM bytes (GB) of one step: see the module docstring."""
    w = np.arange(1, n + 1, dtype=np.float64) ** -exponent
    k = min(budget // (4 * d), n)
    hit = float(w[:k].sum() / w.sum()) if k > 0 else 0.0
    rows = e * (1.0 - hit) * 4 * d
    norms = e * 4 if streamed else e * (1.0 - hit) * 32
    return hit, (rows + n * 4 * d + e * 4 + (n + 1) * 8 + norms) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--edges", type=int, default=100_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--exponent", type=float, default=0.8)
    ap.add_argument("--seed", type=int, default=20240922)   # bench.py's default
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--budgets-mb", default="0,8,16,24,32,40,48,64")
    ap.add_argument("--json", default=None, help="also write the rows as JSON to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("l2_sweep.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, e, d = args.nodes, args.edges, args.dim

    edges = bench.gen_edges(torch, n, e, args.exponent, args.seed, dev)
    indeg = torch.bincount(edges[:, 1], minlength=n)
    norm = ops.degree_norm(indeg).reshape(-1)
    g = pgl.Graph(edges=edges, num_nodes=n)
    fwd = g._fwd_csr()
    del edges, indeg
    x = bench.gen_features(torch, n, d, args.seed + 1, dev)
    out = torch.empty(n, d, device=dev)
    fwd["slot_scale"](norm)
    assert fwd["slot_scale"](norm) is not None     # the second call materialises the per-slot norms

    variants = []
    for mb in (float(v) for v in args.budgets_mb.split(",")):
        pk = tuple(ops.pack_cols(fwd["cols"], n, 4 * d, budget_bytes=int(mb * (1 << 20))))
        variants.append((mb, False, pk))                                        # plain tuple: norm gathered
        variants.append((mb, True, ops.PackedCols(pk, fwd["slot_scale"])))     # norm streamed per slot

    def step(packed):
        return ops._spmm_raw(fwd["indptr"], fwd["cols"], x, n, "sum", scale_src=norm, scale_dst=norm,
                             max_degree=fwd["max_degree"], out=out, packed=packed)

    times = [[] for _ in variants]
    ref = None
    identical = [True] * len(variants)
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for rnd in range(args.rounds):
        order = list(range(len(variants)))
        order = order[rnd % len(order):] + order[:rnd % len(order)]
        for i in order:
            packed = variants[i][2]
            step(packed)                      # warm-up of this variant (and its L2 contents)
            torch.cuda.synchronize()
            for a, b in evs:
                a.record()
                step(packed)
                b.record()
            torch.cuda.synchronize()
            times[i] += [a.elapsed_time(b) for a, b in evs]
            if rnd == 0:
                if ref is None:
                    ref = out.clone()
                else:
                    identical[i] = bool(torch.equal(out, ref))

    info = gpu_info()
    l2 = torch.cuda.get_device_properties(dev).L2_cache_size
    print("# %s | L2 %.1f MB | cfg5 %d nodes / %d edges, %d-d | %d rounds x %d steps per variant"
          % (info, l2 / (1 << 20), n, e, d, args.rounds, args.steps))
    print("%9s %8s %6s %9s %9s %9s %9s %10s %9s %6s" % ("budget_MB", "norm", "hints", "median_ms", "p10_ms", "p90_ms",
                                                       "model_hit", "model_GB", "model_TBs", "same"))
    rows = []
    for (mb, streamed, pk), t, same in zip(variants, times, identical):
        t = np.sort(np.asarray(t))
        med = float(np.median(t))
        hit, gb = model_gb(n, e, d, args.exponent, int(mb * (1 << 20)), streamed)
        row = {"budget_mb": mb, "norm": "streamed" if streamed else "gathered", "hints": bool(pk[1]),
               "median_ms": med, "p10_ms": float(t[len(t) // 10]), "p90_ms": float(t[(len(t) * 9) // 10]),
               "min_ms": float(t[0]), "max_ms": float(t[-1]), "model_hot_share": hit, "model_dram_gb": gb,
               "model_tbs_at_median": gb / med, "identical_to_first": same}
        rows.append(row)
        print("%9.0f %8s %6s %9.3f %9.3f %9.3f %9.2f %10.1f %9.2f %6s" % (
            mb, row["norm"], row["hints"], med, row["p10_ms"], row["p90_ms"], hit, gb, gb / med, same))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "l2_bytes": l2, "nodes": n, "edges": e, "dim": d, "rounds": args.rounds,
                       "steps": args.steps, "rows": rows}, f, indent=1)
    if not all(identical):
        raise SystemExit("l2_sweep.py: a variant's output differs from the first variant's")


if __name__ == "__main__":
    main()
