"""The GCN aggregation step in float32, bfloat16 and float16, alternating inside every round.

Builds bench.py's cfg5 graph once (its own generators: Chung-Lu exponent 0.8, 10M nodes / 100M edges, 128-d) and times
ops._spmm_raw -- both norm scalings, per-slot norms streamed, packed ids with the device's L2 hot budget chosen for the
dtype's row size -- for each dtype.  Every 16-bit output is compared bit for bit, on the full output, with the fp32
step on the widened features rounded to the same dtype: both run the same task plan, so they must be equal.  Then
GCNConv(128, 128) forward + backward is timed in fp32 and under bf16 autocast (fp32 input features, as autocast leaves
them, and bf16 input features).

    python scripts/bench_half.py [--rounds 5] [--steps 10] [--json FILE]

Byte model of one aggregation step (algorithmic bytes: every row gather reaches memory once):
    B = E (b D + 8) + N b D + (N + 1) 8 + 2 N 4,   b = bytes per element (4 or 2)
i.e. row gathers and packed ids / per-slot norms, the output, indptr and the two norm vectors.
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

HBM_TBS = 3.35  # H100 SXM data sheet


def gpu_info():
    """Name, power limit and max SM clock: a read-only nvidia-smi query."""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi failed"
    except (OSError, subprocess.TimeoutExpired) as ex:
        return "nvidia-smi unavailable: %r" % (ex,)


def model_gb(n, e, d, b):
    return (e * (b * d + 8) + n * b * d + (n + 1) * 8 + 2 * n * 4) / 1e9


def stats(t):
    t = np.sort(np.asarray(t))
    return float(np.median(t)), float(t[len(t) // 10]), float(t[(len(t) * 9) // 10])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nodes", type=int, default=10_000_000)
    ap.add_argument("--edges", type=int, default=100_000_000)
    ap.add_argument("--dim", type=int, default=128)
    ap.add_argument("--exponent", type=float, default=0.8)
    ap.add_argument("--seed", type=int, default=20240922)   # bench.py's default
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--layer-steps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results as JSON to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_half.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, e, d = args.nodes, args.edges, args.dim

    edges = bench.gen_edges(torch, n, e, args.exponent, args.seed, dev)
    indeg = torch.bincount(edges[:, 1], minlength=n)
    norm = ops.degree_norm(indeg).reshape(-1)
    g = pgl.Graph(edges=edges, num_nodes=n)
    fwd = g._fwd_csr()
    del edges, indeg
    x32 = bench.gen_features(torch, n, d, args.seed + 1, dev)
    fwd["slot_scale"](norm)
    assert fwd["slot_scale"](norm) is not None     # the second call materialises the per-slot norms

    dtypes = [torch.float32, torch.bfloat16, torch.float16]
    xs = {dt: x32 if dt == torch.float32 else x32.to(dt) for dt in dtypes}
    outs = {dt: torch.empty(n, d, device=dev, dtype=dt) for dt in dtypes}
    packs = {dt: ops.PackedCols(tuple(ops.pack_cols(fwd["cols"], n, d * xs[dt].element_size())), fwd["slot_scale"])
             for dt in dtypes}

    def step(dt, x=None, out=None):
        return ops._spmm_raw(fwd["indptr"], fwd["cols"], xs[dt] if x is None else x, n, "sum", scale_src=norm,
                             scale_dst=norm, max_degree=fwd["max_degree"], out=outs[dt] if out is None else out,
                             packed=packs[dt])

    # bit check on the full output: round16(fp32 step on the widened 16-bit features)
    identical = {}
    ref = torch.empty(n, d, device=dev)
    for dt in dtypes[1:]:
        step(dt)
        step(torch.float32, x=xs[dt].float(), out=ref)
        identical[str(dt)] = bool(torch.equal(outs[dt].view(torch.int16), ref.to(dt).view(torch.int16)))
    del ref

    times = {dt: [] for dt in dtypes}
    pair_faster = {dt: [] for dt in dtypes[1:]}
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for rnd in range(args.rounds):
        order = dtypes[rnd % 3:] + dtypes[:rnd % 3]
        med = {}
        for dt in order:
            step(dt)                      # warm-up of this variant (and its L2 contents)
            torch.cuda.synchronize()
            for a, b in evs:
                a.record()
                step(dt)
                b.record()
            torch.cuda.synchronize()
            t = [a.elapsed_time(b) for a, b in evs]
            times[dt] += t
            med[dt] = float(np.median(t))
        for dt in dtypes[1:]:
            pair_faster[dt].append(med[dt] < med[torch.float32])

    # GCNConv(128, 128) forward + backward
    conv = pgl.nn.GCNConv(d, d).to(dev)
    layer_cases = {"fp32": (torch.float32, False), "autocast_bf16_fp32_input": (torch.float32, True),
                   "autocast_bf16_bf16_input": (torch.bfloat16, True)}
    layer_times = {k: [] for k in layer_cases}
    for rnd in range(args.rounds):
        for name, (in_dt, ac) in layer_cases.items():
            x = xs[in_dt].detach().requires_grad_()

            def fb():
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=ac):
                    out = conv(g, x, norm=norm.reshape(-1, 1))
                out.float().sum().backward()
                x.grad = None
                conv.zero_grad(set_to_none=True)
            fb()
            torch.cuda.synchronize()
            for _ in range(args.layer_steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fb()
                b.record()
                torch.cuda.synchronize()
                layer_times[name].append(a.elapsed_time(b))

    info = gpu_info()
    print("# %s | cfg5 %d nodes / %d edges, %d-d | %d rounds x %d steps per dtype, dtypes alternate in each round"
          % (info, n, e, d, args.rounds, args.steps))
    print("%9s %9s %9s %9s %9s %9s %12s %10s %s" % ("dtype", "median_ms", "p10_ms", "p90_ms", "Gedge_s", "model_GB",
                                                   "model_ms@3.35", "faster", "bits"))
    rows = []
    for dt in dtypes:
        med, p10, p90 = stats(times[dt])
        gb = model_gb(n, e, d, xs[dt].element_size())
        row = {"dtype": str(dt), "median_ms": med, "p10_ms": p10, "p90_ms": p90, "gedges_per_s": e / med / 1e6,
               "model_gb": gb, "model_ms_at_datasheet_bw": gb / HBM_TBS,
               "faster_than_fp32_in_pairs": pair_faster.get(dt), "bit_identical_to_rounded_fp32": identical.get(str(dt))}
        rows.append(row)
        faster = "-" if dt == torch.float32 else "%d/%d" % (sum(pair_faster[dt]), len(pair_faster[dt]))
        bits = "-" if dt == torch.float32 else ("identical" if identical[str(dt)] else "DIFFERENT")
        print("%9s %9.3f %9.3f %9.3f %9.2f %9.1f %12.2f %10s %s" % (str(dt).replace("torch.", ""), med, p10, p90,
                                                                   row["gedges_per_s"], gb, gb / HBM_TBS, faster, bits))
    print("%26s %9s %9s %9s" % ("GCNConv(128,128) fwd+bwd", "median_ms", "p10_ms", "p90_ms"))
    layer_rows = {}
    for name, t in layer_times.items():
        med, p10, p90 = stats(t)
        layer_rows[name] = {"median_ms": med, "p10_ms": p10, "p90_ms": p90}
        print("%26s %9.3f %9.3f %9.3f" % (name, med, p10, p90))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "nodes": n, "edges": e, "dim": d, "rounds": args.rounds, "steps": args.steps,
                       "aggregation": rows, "gcnconv": layer_rows}, f, indent=1)
    if not all(identical.values()):
        raise SystemExit("bench_half.py: a 16-bit output differs from the rounded fp32 output")


if __name__ == "__main__":
    main()
