"""cfg3's GATv2Conv on the fused GATv2 attention against the op-by-op route, alternating inside every round.

Builds bench_gat.py's cfg3 graph (RMAT scale 20, 10M edges) and, for GATv2Conv(128 -> 8 heads x 16) and
GATv2Conv(64 -> 8 heads x 8) in float32 and bfloat16, times
  * inference forward (no_grad, eval) and training forward + backward with attn_drop 0 and 0.6, each through the layer
    (which takes ops.gatv2_attention) and through the op-by-op route restated below (send_uv(add) + LeakyReLU + the
    product with attn + sum + edge_softmax + dropout + send_ue_recv, the layer's route for the shapes the kernels
    refuse);
  * the three new kernels alone: the forward entry (inference, no lse), the edge backward entry (with grad attn) and
    the score-gradient aggregation over the dst-keyed CSR;
  * the peak memory of one training step (p = 0) on either route.
Before timing, the fused layer's output is checked against the op-by-op one on the full graph.

    python scripts/bench_gatv2.py [--rounds 3] [--steps 10] [--layer-steps 3] [--json FILE]

Byte model of the forward kernel (algorithmic bytes: every gathered row reaches memory once):
    B = E (8 + b D) + N (2 b D + 4 H) + (N + 1) 8,   b = bytes per element (4 or 2)
i.e. per edge the column id and the source's feature row, per row f[d], out, lse and the row pointer.
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
import pgl_b200.nn.functional as GF  # noqa: E402
from bench_gat import rmat  # noqa: E402
from bench_half import HBM_TBS, gpu_info, stats  # noqa: E402
from pgl_b200 import ops  # noqa: E402


def model_gb(n, e, d, h, b):
    return (e * (8 + b * d) + n * (2 * b * d + 4 * h) + (n + 1) * 8) / 1e9


def op_by_op(conv, g, x):
    """GATv2Conv.forward on the op-by-op route."""
    H, Dh = conv.num_heads, conv.hidden_size
    feature = conv.linear(x).reshape(-1, H, Dh)
    alpha = conv.leaky_relu(g.send_uv(feature, feature, "add"))
    alpha = GF.edge_softmax(g, torch.sum(alpha * conv.attn, dim=-1)).reshape(-1, H, 1)
    if conv.attn_drop > 1e-15:
        alpha = conv.attn_dropout(alpha)
    return g.send_ue_recv(feature, alpha, "mul", "sum").reshape(-1, H * Dh)


def peak_gb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 1e9


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
        raise SystemExit("bench_gatv2.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, e = 1 << args.scale, args.edges
    g = pgl.Graph(edges=rmat(args.scale, e), num_nodes=n)
    fwd, bwd = g._fwd_csr(), g._bwd_csr()
    info = gpu_info()
    print("# %s | cfg3 RMAT scale %d, %d edges | %d rounds, fused and op-by-op alternate in each round"
          % (info, args.scale, e, args.rounds))
    results = []
    slope = 0.2
    for din, Dh in ((128, 16), (64, 8)):
        H = 8
        D = H * Dh
        for dt in (torch.float32, torch.bfloat16):
            torch.manual_seed(2)
            conv = pgl.nn.GATv2Conv(din, Dh, feat_drop=0.0, attn_drop=0.0, num_heads=H).to(dev).to(dt)
            x = torch.randn(n, din, device=dev).to(dt)
            with torch.no_grad():
                conv.eval()
                got, want = conv(g, x), op_by_op(conv, g, x)
                err = float((got.double() - want.double()).abs().max() / want.double().abs().max())
                f2 = conv.linear(x).reshape(n, D).contiguous()
                a32 = conv.attn.detach().reshape(D).float().contiguous()
                del got, want
            out, lse = ops._gatv2_fwd_raw(fwd, f2, a32, slope, H, Dh, None, True)
            go = torch.randn(n, D, device=dev).to(dt)
            beta = torch.empty((e, H), device=dev)
            ds = torch.empty((e, H), device=dev)
            ga = torch.empty((D,), device=dev)
            gr = torch.empty((n, D), device=dev)
            need = ops.ctypes.c_size_t(0)
            ops.check(ops.lib.pglb_gatv2_bwd_edge_ws(e, ops.ctypes.byref(need)))
            ws_e = torch.empty(need.value, dtype=torch.uint8, device=dev)
            ops.check(ops.lib.pglb_spmm_csr_ws(n, e, D, ops.ctypes.byref(need)))
            ws_a = torch.empty(need.value, dtype=torch.uint8, device=dev)
            half = dt != torch.float32
            dtc = (ops._DTYPE16[dt],) if half else ()
            bwd_entry = ops.lib.pglb_gatv2_bwd_edge_x16 if half else ops.lib.pglb_gatv2_bwd_edge_f32
            score_entry = ops.lib.pglb_gatv2_score_grad_x16 if half else ops.lib.pglb_gatv2_score_grad_f32

            def k_fwd():
                ops._gatv2_fwd_raw(fwd, f2, a32, slope, H, Dh, None, False)

            def k_bwd():
                ops.check(bwd_entry(ops._ptr(fwd["rows"]), ops._ptr(fwd["cols"]), ops._ptr(fwd["eid"]), ops._ptr(f2), D,
                                    ops._ptr(a32), slope, ops._ptr(go), D, ops._ptr(out), D, ops._ptr(lse), e, H, Dh,
                                    *dtc, ops._ptr(beta), ops._ptr(ds), ops._ptr(ga), ops._ptr(ws_e), ws_e.numel(),
                                    ops._stream()))

            def k_score():
                ops.check(score_entry(ops._ptr(fwd["indptr"]), ops._ptr(fwd["cols"]), ops._ptr(fwd["eid"]),
                                      ops._ptr(f2), D, ops._ptr(a32), slope, ops._ptr(ds), ops._ptr(gr), D, n, e, H, Dh,
                                      *dtc, 0, ops._ptr(ws_a), ws_a.numel(), ops._stream()))

            def infer(fused):
                def f():
                    with torch.no_grad():
                        conv.eval()
                        return conv(g, x) if fused else op_by_op(conv, g, x)
                return f

            def train(fused, p):
                def f():
                    conv.train()
                    conv.attn_drop = p
                    conv.attn_dropout.p = p
                    xin = x.detach().requires_grad_()
                    o = conv(g, xin) if fused else op_by_op(conv, g, xin)
                    o.float().sum().backward()
                    conv.zero_grad(set_to_none=True)
                return f

            k_bwd()
            peaks = {"fused_train_peak_gb": peak_gb(train(True, 0.0)),
                     "op_by_op_train_peak_gb": peak_gb(train(False, 0.0))}
            cases = {"kernel_fwd": (k_fwd, None), "kernel_bwd_edge": (k_bwd, None),
                     "kernel_score_grad": (k_score, None),
                     "infer": (infer(True), infer(False)),
                     "train_p0": (train(True, 0.0), train(False, 0.0)),
                     "train_p0.6": (train(True, 0.6), train(False, 0.6))}
            times = {name: ([], []) for name in cases}
            faster = {name: [] for name in cases}
            for rnd in range(args.rounds):
                for name, (fu, ob) in cases.items():
                    steps = args.steps if name.startswith("kernel") else args.layer_steps
                    pair = [(0, fu), (1, ob)] if ob is not None else [(0, fu)]
                    if rnd % 2:
                        pair.reverse()
                    med = {}
                    for i, fn in pair:
                        t = timed(fn, steps)
                        times[name][i].extend(t)
                        med[i] = float(np.median(t))
                    if ob is not None:
                        faster[name].append(med[0] < med[1])
            conv.attn_drop = 0.0
            tag = "GATv2Conv(%d -> %d x %d) %s" % (din, H, Dh, str(dt).replace("torch.", ""))
            print("# %s: fused vs op-by-op output, max |diff| / max |ref| = %.2e" % (tag, err))
            print("# %s: training peak memory, fused %.2f GB, op-by-op %.2f GB" % (
                tag, peaks["fused_train_peak_gb"], peaks["op_by_op_train_peak_gb"]))
            print("%-17s %10s %8s %8s %12s %8s %8s %8s %8s" % ("case", "fused_ms", "p10", "p90", "op_by_op_ms", "p10",
                                                                 "p90", "speedup", "faster"))
            row = {"layer": tag, "output_rel_err": err, "cases": {}, **peaks}
            for name in cases:
                fm, f10, f90 = stats(times[name][0])
                entry = {"fused_median_ms": fm, "fused_p10_ms": f10, "fused_p90_ms": f90}
                if times[name][1]:
                    om, o10, o90 = stats(times[name][1])
                    entry.update({"op_by_op_median_ms": om, "op_by_op_p10_ms": o10, "op_by_op_p90_ms": o90,
                                  "fused_faster_in_rounds": faster[name]})
                    print("%-17s %10.3f %8.3f %8.3f %12.3f %8.3f %8.3f %7.2fx %6d/%d" % (
                        name, fm, f10, f90, om, o10, o90, om / fm, sum(faster[name]), len(faster[name])))
                else:
                    extra = ""
                    if name == "kernel_fwd":
                        gb = model_gb(n, e, D, H, x.element_size())
                        entry.update({"model_gb": gb, "achieved_tbs": gb / fm, "fraction_of_3.35_tbs": gb / fm / HBM_TBS})
                        extra = "  model %.3f GB, %.2f TB/s = %.0f%% of %.2f TB/s" % (gb, gb / fm, 100 * gb / fm / HBM_TBS,
                                                                                  HBM_TBS)
                    print("%-17s %10.3f %8.3f %8.3f%s" % (name, fm, f10, f90, extra))
                row["cases"][name] = entry
            results.append(row)
            del conv, x, f2, out, lse, go, beta, ds, gr, ws_e, ws_a
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "nodes": n, "edges": e, "rounds": args.rounds, "results": results}, f, indent=1)
    if any(r["output_rel_err"] > (1e-4 if "float32" in r["layer"] else 3e-2) for r in results):
        raise SystemExit("bench_gatv2.py: the fused output differs from the op-by-op output")


if __name__ == "__main__":
    main()
