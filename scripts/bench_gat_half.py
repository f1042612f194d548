"""cfg3's GAT aggregation and GATConv layer in float32, bfloat16 and float16, alternating inside every round.

Builds bench_gat.py's cfg3 graph (RMAT scale 20, 10M edges) and GATConv(128 -> 8 heads x 16), then times
  * the fused inference aggregation ops.gat_fused with f in each dtype (float32 attention, result in f's dtype);
  * GATConv forward + backward for an fp32 module, a bf16 and an fp16 module (the fused 16-bit training path), and a
    bf16 module on the op-by-op route (ops.GAT_FUSED_TRAIN = False: send_uv + LeakyReLU + edge_softmax +
    send_ue_recv, the route every 16-bit GATConv took before the 16-bit GAT kernels).
Every 16-bit fused output (the aggregation and the training forward on the same inputs) is compared bit for bit, on
the full output, with the fp32 kernel's output on the widened features rounded to the same dtype, in every round.

    python scripts/bench_gat_half.py [--rounds 5] [--steps 20] [--layer-steps 5] [--json FILE]

Byte model of one aggregation (algorithmic bytes: every gathered row reaches memory once):
    B = E (b D + 4 H + 8) + N (b D + 4 H) + (N + 1) 8,   b = bytes per feature element (4 or 2)
i.e. per edge the source's feature row, its attention row and the column id, per node the output row and attn_dst.
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
from bench_half import HBM_TBS, gpu_info, stats  # noqa: E402
from pgl_b200 import ops  # noqa: E402


def model_gb(n, e, d, h, b):
    return (e * (b * d + 4 * h + 8) + n * (b * d + 4 * h) + (n + 1) * 8) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=20)
    ap.add_argument("--edges", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--layer-steps", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the results as JSON to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gat_half.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, e, H, Dh = 1 << args.scale, args.edges, 8, 16
    D = H * Dh
    g = pgl.Graph(edges=rmat(args.scale, e), num_nodes=n)
    csr = g._fwd_csr()
    g._bwd_csr()
    torch.manual_seed(2)
    x = torch.randn(n, 128, device=dev)
    conv = pgl.nn.GATConv(128, Dh, feat_drop=0, attn_drop=0, num_heads=H).to(dev)
    with torch.no_grad():
        f32 = (x @ conv.linear.weight + conv.linear.bias).reshape(-1, H, Dh)
        a_s = (f32 * conv.weight_src).sum(-1)
        a_d = (f32 * conv.weight_dst).sum(-1)
    dtypes = [torch.float32, torch.bfloat16, torch.float16]
    fs = {dt: f32 if dt == torch.float32 else f32.to(dt) for dt in dtypes}

    def agg(dt):
        return ops.gat_fused(csr, fs[dt], a_s, a_d, 0.2, out_dtype=dt)

    # aggregation: alternating dtypes, bit check of every 16-bit output in every round
    times = {dt: [] for dt in dtypes}
    pair_faster = {dt: [] for dt in dtypes[1:]}
    identical = {str(dt): True for dt in dtypes[1:]}
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    with torch.no_grad():
        for rnd in range(args.rounds):
            order = dtypes[rnd % 3:] + dtypes[:rnd % 3]
            med = {}
            for dt in order:
                out = agg(dt)                      # warm-up of this variant
                if dt != torch.float32:
                    ref = ops.gat_fused(csr, fs[dt].float(), a_s, a_d, 0.2).to(dt)
                    identical[str(dt)] &= bool(torch.equal(out.view(torch.int16), ref.view(torch.int16)))
                    # the training forward (the same kernel, which also writes lse)
                    tr = ops.gat_fused_train(csr, g._bwd_csr, fs[dt], a_s, a_d, 0.2, out_dtype=dt)
                    identical["train_" + str(dt)] = identical.get("train_" + str(dt), True) and bool(
                        torch.equal(tr.view(torch.int16), ref.view(torch.int16)))
                    del ref, tr
                torch.cuda.synchronize()
                for a, b in evs:
                    a.record()
                    agg(dt)
                    b.record()
                torch.cuda.synchronize()
                t = [a.elapsed_time(b) for a, b in evs]
                times[dt] += t
                med[dt] = float(np.median(t))
            for dt in dtypes[1:]:
                pair_faster[dt].append(med[dt] < med[torch.float32])

    # GATConv forward + backward
    mods = {}
    for name, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16), ("fp16", torch.float16),
                     ("bf16_op_by_op", torch.bfloat16)):
        m = pgl.nn.GATConv(128, Dh, feat_drop=0, attn_drop=0, num_heads=H).to(dev)
        m.load_state_dict(conv.state_dict())
        mods[name] = (m.to(dt), dt, name != "bf16_op_by_op")
    layer_times = {k: [] for k in mods}
    layer_pair_faster = {k: [] for k in mods if k != "fp32"}
    for rnd in range(args.rounds):
        names = list(mods)
        order = names[rnd % len(names):] + names[:rnd % len(names)]
        med = {}
        for name in order:
            m, dt, fused = mods[name]
            xin = x.to(dt).requires_grad_()

            def fb():
                out = m(g, xin)
                out.float().sum().backward()
                xin.grad = None
                m.zero_grad(set_to_none=True)
                return out
            old = ops.GAT_FUSED_TRAIN
            ops.GAT_FUSED_TRAIN = fused
            try:
                fb()
                torch.cuda.synchronize()
                t = []
                for _ in range(args.layer_steps):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    fb()
                    b.record()
                    torch.cuda.synchronize()
                    t.append(a.elapsed_time(b))
            finally:
                ops.GAT_FUSED_TRAIN = old
            layer_times[name] += t
            med[name] = float(np.median(t))
        for name in layer_pair_faster:
            ref_name = "bf16_op_by_op" if name.startswith("bf16") and name != "bf16_op_by_op" else "fp32"
            layer_pair_faster[name].append(med[name] < med[ref_name])

    info = gpu_info()
    print("# %s | cfg3 RMAT scale %d, %d edges, GATConv(128 -> %d x %d) | %d rounds, dtypes alternate in each round"
          % (info, args.scale, e, H, Dh, args.rounds))
    print("%9s %9s %9s %9s %9s %13s %10s %s" % ("dtype", "median_ms", "p10_ms", "p90_ms", "model_GB", "model_ms@3.35",
                                               "faster", "bits"))
    rows = []
    for dt in dtypes:
        med, p10, p90 = stats(times[dt])
        gb = model_gb(n, e, D, H, fs[dt].element_size())
        row = {"dtype": str(dt), "median_ms": med, "p10_ms": p10, "p90_ms": p90, "model_gb": gb,
               "model_ms_at_datasheet_bw": gb / HBM_TBS, "faster_than_fp32_in_pairs": pair_faster.get(dt),
               "bit_identical_to_rounded_fp32": identical.get(str(dt))}
        rows.append(row)
        faster = "-" if dt == torch.float32 else "%d/%d" % (sum(pair_faster[dt]), len(pair_faster[dt]))
        bits = "-" if dt == torch.float32 else ("identical" if identical[str(dt)] else "DIFFERENT")
        print("%9s %9.3f %9.3f %9.3f %9.3f %13.3f %10s %s" % (str(dt).replace("torch.", ""), med, p10, p90, gb,
                                                            gb / HBM_TBS, faster, bits))
    print("# 16-bit training forward on the same inputs: %s" % ", ".join(
        "%s %s" % (k[6:].replace("torch.", ""), "identical" if v else "DIFFERENT")
        for k, v in identical.items() if k.startswith("train_")))
    print("%30s %9s %9s %9s %14s" % ("GATConv fwd+bwd", "median_ms", "p10_ms", "p90_ms", "faster"))
    layer_rows = {}
    for name, t in layer_times.items():
        med, p10, p90 = stats(t)
        fp = layer_pair_faster.get(name)
        vs = "" if fp is None else ("%d/%d vs %s" % (sum(fp), len(fp), "op-by-op" if name == "bf16" else "fp32"))
        layer_rows[name] = {"median_ms": med, "p10_ms": p10, "p90_ms": p90, "faster_in_pairs": fp}
        print("%30s %9.3f %9.3f %9.3f %14s" % (name, med, p10, p90, vs))
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "nodes": n, "edges": e, "heads": H, "head_dim": Dh, "rounds": args.rounds,
                       "aggregation": rows, "bit_identical": identical, "gatconv_fwd_bwd": layer_rows}, f, indent=1)
    if not all(identical.values()):
        raise SystemExit("bench_gat_half.py: a 16-bit output differs from the rounded fp32 output")


if __name__ == "__main__":
    main()
