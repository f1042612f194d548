"""cfg3's TransformerConv WITH edge features on the fused dot-product attention against the op-by-op route (the layer's
graph.send / graph.recv pair), alternating inside every round.

Builds bench_gat.py's cfg3 graph (RMAT scale 20, 10M edges) and, for TransformerConv(128 -> 8 heads x 16) and
TransformerConv(64 -> 8 heads x 8) in float32 and bfloat16 with edge features [E, H*Dh], times
  * the two kernels alone: the forward entry (inference, no lse) and the edge backward entry (with grad_e);
  * inference forward (no_grad, eval) and training forward + backward (edge features requiring a gradient) with
    attn_drop 0 and 0.6, each through the layer (ops.dot_attention) and through the op-by-op route;
and reports the forward + backward peak memory above the resident inputs for both routes.  Before timing, the fused
layer's output is checked against the op-by-op one on the full graph.  An op-by-op case that runs out of memory is
recorded as such ("oom"); --scale / --edges select a smaller RMAT graph to compare on.

    python scripts/bench_transformer_edge.py [--scale 20] [--edges 10000000] [--rounds 3] [--steps 10]
                                             [--layer-steps 3] [--json FILE]

Byte model of the forward kernel (algorithmic bytes: every gathered row reaches memory once):
    B = E (16 + 3 b D) + N (2 b D + 4 H) + (N + 1) 8,   b = bytes per element (4 or 2)
i.e. per edge the column id, the edge id and the k, v and e rows, per row q, out, lse and the row pointer.
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
from pgl_b200 import ops  # noqa: E402


def model_gb(n, e, d, h, b):
    return (e * (16 + 3 * b * d) + n * (2 * b * d + 4 * h) + (n + 1) * 8) / 1e9


def op_by_op(conv, g, x, ef):
    """conv(g, x, ef) with ops.dot_attention declining: the layer's send / recv route."""
    real = ops.dot_attention
    ops.dot_attention = lambda *a, **kw: None
    try:
        return conv(g, x, ef)
    finally:
        ops.dot_attention = real


def timed(fn, steps):
    fn()
    torch.cuda.synchronize()
    t = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        t.append(a.elapsed_time(b))
    return t


def peak_gb(fn):
    """Peak memory of one call above what was allocated before it, in GB; None when it runs out of memory."""
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    try:
        fn()
        torch.cuda.synchronize()
    except torch.cuda.OutOfMemoryError:
        torch.cuda.empty_cache()
        return None
    return (torch.cuda.max_memory_allocated() - base) / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=20)
    ap.add_argument("--edges", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--layer-steps", type=int, default=3)
    ap.add_argument("--json", default=None, help="also write the results as JSON to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_transformer_edge.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, e = 1 << args.scale, args.edges
    g = pgl.Graph(edges=rmat(args.scale, e), num_nodes=n)
    fwd, bwd = g._fwd_csr(), g._bwd_csr()
    info = gpu_info()
    print("# %s | RMAT scale %d, %d edges | %d rounds, fused and op-by-op alternate in each round"
          % (info, args.scale, e, args.rounds))
    results = []
    for din, Dh in ((128, 16), (64, 8)):
        H = 8
        D = H * Dh
        for dt in (torch.float32, torch.bfloat16):
            torch.manual_seed(2)
            conv = pgl.nn.TransformerConv(din, Dh, num_heads=H, feat_drop=0.0, attn_drop=0.0).to(dev).to(dt)
            x = torch.randn(n, din, device=dev).to(dt)
            ef = (0.5 * torch.randn(e, D, device=dev)).to(dt)
            tag = "TransformerConv(%d -> %d x %d) %s" % (din, H, Dh, str(dt).replace("torch.", ""))
            with torch.no_grad():
                conv.eval()
                got = conv(g, x, ef)
                try:
                    want = op_by_op(conv, g, x, ef)
                    err = float((got.double() - want.double()).abs().max() / want.double().abs().max())
                    del want
                except torch.cuda.OutOfMemoryError:
                    err = None
                    torch.cuda.empty_cache()
                del got
                q = (conv.q(x).reshape(-1, H, Dh) / Dh ** 0.5).reshape(n, D).contiguous()
                k = conv.k(x).reshape(n, D).contiguous()
                v = conv.v(x).reshape(n, D).contiguous()
            out, lse = ops._dot_attn_fwd_raw(fwd, q, k, v, H, Dh, None, True, ef)
            go = torch.randn(n, D, device=dev).to(dt)
            beta = torch.empty((e, H), device=dev)
            ds = torch.empty((e, H), device=dev)
            ge = torch.empty_like(ef)
            half = dt != torch.float32
            dtc = (ops._DTYPE16[dt],) if half else ()
            bwd_entry = ops.lib.pglb_dot_attn_e_bwd_edge_x16 if half else ops.lib.pglb_dot_attn_e_bwd_edge_f32

            def k_fwd():
                ops._dot_attn_fwd_raw(fwd, q, k, v, H, Dh, None, False, ef)

            def k_bwd():
                ops.check(bwd_entry(ops._ptr(fwd["rows"]), ops._ptr(fwd["cols"]), ops._ptr(fwd["eid"]), ops._ptr(q), D,
                                    ops._ptr(k), D, ops._ptr(v), D, ops._ptr(ef), D, ops._ptr(go), D, ops._ptr(out), D,
                                    ops._ptr(lse), e, H, Dh, *dtc, ops._ptr(beta), ops._ptr(ds), ops._ptr(ge), D,
                                    ops._stream()))

            def infer(fused):
                def f():
                    with torch.no_grad():
                        conv.eval()
                        return conv(g, x, ef) if fused else op_by_op(conv, g, x, ef)
                return f

            def train(fused, p):
                def f():
                    conv.train()
                    conv.attn_drop = p
                    conv.attn_dropout.p = p
                    xin = x.detach().requires_grad_()
                    ein = ef.detach().requires_grad_()
                    o = conv(g, xin, ein) if fused else op_by_op(conv, g, xin, ein)
                    o.float().sum().backward()
                    conv.zero_grad(set_to_none=True)
                return f

            peak = {"fused_gb": peak_gb(train(True, 0.0)), "op_by_op_gb": peak_gb(train(False, 0.0))}
            cases = {"kernel_fwd": (k_fwd, None), "kernel_bwd_edge": (k_bwd, None),
                     "infer": (infer(True), infer(False)),
                     "train_p0": (train(True, 0.0), train(False, 0.0)),
                     "train_p0.6": (train(True, 0.6), train(False, 0.6))}
            times = {name: ([], []) for name in cases}
            faster = {name: [] for name in cases}
            oom = set()
            for rnd in range(args.rounds):
                for name, (fu, ob) in cases.items():
                    steps = args.steps if name.startswith("kernel") else args.layer_steps
                    pair = [(0, fu), (1, ob)] if ob is not None else [(0, fu)]
                    if rnd % 2:
                        pair.reverse()
                    med = {}
                    for i, fn in pair:
                        if i == 1 and name in oom:
                            continue
                        try:
                            t = timed(fn, steps)
                        except torch.cuda.OutOfMemoryError:
                            if i == 0:
                                raise
                            oom.add(name)
                            torch.cuda.empty_cache()
                            continue
                        times[name][i].extend(t)
                        med[i] = float(np.median(t))
                    if ob is not None and 1 in med:
                        faster[name].append(med[0] < med[1])
            conv.attn_drop = 0.0
            print("# %s: fused vs op-by-op output, max |diff| / max |ref| = %s" %
                  (tag, "op-by-op out of memory" if err is None else "%.2e" % err))
            print("# %s: forward + backward peak above the inputs: fused %s GB, op-by-op %s GB" % (
                tag, "%.3f" % peak["fused_gb"], "oom" if peak["op_by_op_gb"] is None else "%.3f" % peak["op_by_op_gb"]))
            print("%-16s %10s %8s %8s %12s %8s %8s %8s %8s" % ("case", "fused_ms", "p10", "p90", "op_by_op_ms", "p10",
                                                                 "p90", "speedup", "faster"))
            row = {"layer": tag, "output_rel_err": err, "peak_memory": peak, "cases": {}}
            for name in cases:
                fm, f10, f90 = stats(times[name][0])
                entry = {"fused_median_ms": fm, "fused_p10_ms": f10, "fused_p90_ms": f90}
                if name in oom:
                    entry["op_by_op"] = "oom"
                    print("%-16s %10.3f %8.3f %8.3f %12s" % (name, fm, f10, f90, "oom"))
                elif times[name][1]:
                    om, o10, o90 = stats(times[name][1])
                    entry.update({"op_by_op_median_ms": om, "op_by_op_p10_ms": o10, "op_by_op_p90_ms": o90,
                                  "fused_faster_in_rounds": faster[name]})
                    print("%-16s %10.3f %8.3f %8.3f %12.3f %8.3f %8.3f %7.2fx %6d/%d" % (
                        name, fm, f10, f90, om, o10, o90, om / fm, sum(faster[name]), len(faster[name])))
                else:
                    extra = ""
                    if name == "kernel_fwd":
                        gb = model_gb(n, e, D, H, x.element_size())
                        entry.update({"model_gb": gb, "model_tbs": gb / fm})
                        extra = "  model %.3f GB, %.2f TB/s (model bytes / time)" % (gb, gb / fm)
                    print("%-16s %10.3f %8.3f %8.3f%s" % (name, fm, f10, f90, extra))
                row["cases"][name] = entry
            results.append(row)
            del conv, x, ef, q, k, v, out, lse, go, beta, ds, ge
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "nodes": n, "edges": e, "rounds": args.rounds, "results": results}, f, indent=1)
    if any(r["output_rel_err"] is not None and r["output_rel_err"] > (1e-4 if "float32" in r["layer"] else 3e-2)
           for r in results):
        raise SystemExit("bench_transformer_edge.py: the fused output differs from the op-by-op output")


if __name__ == "__main__":
    main()
