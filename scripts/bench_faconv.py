"""cfg3's FAConv on the fused self-gated aggregation against the op-by-op route, alternating inside every round.

Builds bench_gat.py's cfg3 graph (RMAT scale 20, 10M edges) and, for FAConv at D = 16 (the FAGCN example's width), 64
and 128 in float32 and bfloat16, times
  * inference forward (no_grad, eval) and training forward + backward at p = 0 and p = 0.6, each through the layer
    (which takes ops.fa_attention) and through the op-by-op route restated below (send_uv(add) + tanh + the product with
    send_uv(norm, norm, mul) + dropout + send_ue_recv, the layer's route for the calls the kernels refuse), with CUDA
    events, fused and op-by-op alternating in every round;
  * the forward entry (inference) and the edge-backward entry alone, in a separate pass under torch.profiler: the
    device time of every kernel each launches, per call;
  * the peak memory of one training step (p = 0) on either route.
Before timing, the fused layer's output is checked against the op-by-op one on the full graph.  The card name, power
limit and max SM clock are read (nvidia-smi, read-only) in the same run.

    python scripts/bench_faconv.py [--rounds 3] [--layer-steps 3] [--kernel-steps 20] [--json FILE]

Byte model of the forward kernel (algorithmic bytes: every gathered row reaches memory once):
    B = E (8 + b D + 16) + N (16 + b D) + (N + 1) 8,   b = bytes per element (4 or 2)
i.e. per edge the column id, the source's feature row and the source's 16-byte node record (g_src, norm, g_dst, 0);
per row the dst record, the out row and the row pointer.
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


def model_gb(n, e, d, b):
    return (e * (8 + b * d + 16) + n * (16 + b * d) + (n + 1) * 8) / 1e9


def op_by_op(conv, g, x):
    """FAConv.forward on the op-by-op route."""
    norm = GF.degree_norm(g)
    d = conv.hidden_size
    g_src = x @ conv.gate.weight[:d]
    g_dst = x @ conv.gate.weight[d:] + conv.gate.bias
    h = torch.tanh(g.send_uv(g_src, g_dst, "add"))
    alpha = conv.dropout(h * g.send_uv(norm, norm, "mul"))
    return g.send_ue_recv(x, alpha, "mul", "sum")


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


def profiled(fn, steps):
    """{kernel name: device ms per call of fn} over `steps` calls, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            t = getattr(ev, "device_time", None)
            t = getattr(ev, "cuda_time", 0.0) if t is None else t
            per[ev.name] = per.get(ev.name, 0.0) + t / 1000.0 / steps
    return per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=int, default=20)
    ap.add_argument("--edges", type=int, default=10_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layer-steps", type=int, default=3)
    ap.add_argument("--kernel-steps", type=int, default=20)
    ap.add_argument("--dims", default="16,64,128")
    ap.add_argument("--json", default=None, help="also write the results as JSON to this file")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_faconv.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, e = 1 << args.scale, args.edges
    g = pgl.Graph(edges=rmat(args.scale, e), num_nodes=n)
    g.tensor()
    fwd, bwd = g._fwd_csr(), g._bwd_csr()
    norm = GF.degree_norm(g)
    info = gpu_info()
    print("# %s | cfg3 RMAT scale %d, %d edges | %d rounds, fused and op-by-op alternate in each round"
          % (info, args.scale, e, args.rounds))
    results = []
    for D in (int(v) for v in args.dims.split(",")):
        for dt in (torch.float32, torch.bfloat16):
            torch.manual_seed(2)
            conv = pgl.nn.FAConv(D, drop=0.0).to(dev).to(dt)
            x = torch.randn(n, D, device=dev).to(dt)
            with torch.no_grad():
                conv.eval()
                got, want = conv(g, x), op_by_op(conv, g, x)
                err = float((got.double() - want.double()).abs().max() / want.double().abs().max())
                gs = x @ conv.gate.weight[:D]
                gd = x @ conv.gate.weight[D:] + conv.gate.bias
                rec = ops._fa_records(gs.reshape(n), norm.reshape(n), gd.reshape(n))
                del got, want
            go = torch.randn(n, D, device=dev).to(dt)
            beta = torch.empty(e, device=dev)
            dz = torch.empty(e, device=dev)
            half = dt != torch.float32
            dtc = (ops._DTYPE16[dt],) if half else ()
            bwd_entry = ops.lib.pglb_fa_bwd_edge_x16 if half else ops.lib.pglb_fa_bwd_edge_f32

            def k_fwd():
                ops._fa_fwd_raw(fwd, x, rec, None)

            def k_bwd():
                ops.check(bwd_entry(ops._ptr(fwd["rows"]), ops._ptr(fwd["cols"]), ops._ptr(fwd["eid"]), ops._ptr(x), D,
                                    ops._ptr(rec), ops._ptr(go), D, e, D, *dtc, ops._ptr(beta), ops._ptr(dz),
                                    ops._stream()))

            def infer(fused):
                def f():
                    with torch.no_grad():
                        conv.eval()
                        return conv(g, x) if fused else op_by_op(conv, g, x)
                return f

            def train(fused, p):
                def f():
                    conv.train()
                    conv.dropout.p = p
                    xin = x.detach().requires_grad_()
                    o = conv(g, xin) if fused else op_by_op(conv, g, xin)
                    o.float().sum().backward()
                    conv.zero_grad(set_to_none=True)
                return f

            peaks = {"fused_train_peak_gb": peak_gb(train(True, 0.0)),
                     "op_by_op_train_peak_gb": peak_gb(train(False, 0.0))}
            cases = {"infer": (infer(True), infer(False)),
                     "train_p0": (train(True, 0.0), train(False, 0.0)),
                     "train_p0.6": (train(True, 0.6), train(False, 0.6))}
            times = {name: ([], []) for name in cases}
            faster = {name: [] for name in cases}
            for rnd in range(args.rounds):
                for name, (fu, ob) in cases.items():
                    pair = [(0, fu), (1, ob)]
                    if rnd % 2:
                        pair.reverse()
                    med = {}
                    for i, fn in pair:
                        t = timed(fn, args.layer_steps)
                        times[name][i].extend(t)
                        med[i] = float(np.median(t))
                    faster[name].append(med[0] < med[1])
            conv.dropout.p = 0.0
            kernels = {"kernel_fwd": profiled(k_fwd, args.kernel_steps),
                       "kernel_bwd_edge": profiled(k_bwd, args.kernel_steps)}
            tag = "FAConv(%d) %s" % (D, str(dt).replace("torch.", ""))
            print("# %s: fused vs op-by-op output, max |diff| / max |ref| = %.2e" % (tag, err))
            print("# %s: training peak memory, fused %.3f GB, op-by-op %.3f GB" % (
                tag, peaks["fused_train_peak_gb"], peaks["op_by_op_train_peak_gb"]))
            print("%-17s %10s %8s %8s %12s %8s %8s %8s %8s" % ("case", "fused_ms", "p10", "p90", "op_by_op_ms", "p10",
                                                                 "p90", "speedup", "faster"))
            row = {"layer": tag, "output_rel_err": err, "cases": {}, "kernels": {}, **peaks}
            for name in cases:
                fm, f10, f90 = stats(times[name][0])
                om, o10, o90 = stats(times[name][1])
                row["cases"][name] = {"fused_median_ms": fm, "fused_p10_ms": f10, "fused_p90_ms": f90,
                                      "op_by_op_median_ms": om, "op_by_op_p10_ms": o10, "op_by_op_p90_ms": o90,
                                      "fused_faster_in_rounds": faster[name]}
                print("%-17s %10.3f %8.3f %8.3f %12.3f %8.3f %8.3f %7.2fx %6d/%d" % (
                    name, fm, f10, f90, om, o10, o90, om / fm, sum(faster[name]), len(faster[name])))
            for name, per in kernels.items():
                total = sum(per.values())
                entry = {"device_ms_per_call": total, "per_kernel_ms": per}
                extra = ""
                if name == "kernel_fwd":
                    gb = model_gb(n, e, D, x.element_size())
                    entry.update({"model_gb": gb, "achieved_tbs": gb / total,
                                  "fraction_of_3.35_tbs": gb / total / HBM_TBS})
                    extra = "  model %.3f GB, %.2f TB/s = %.0f%% of %.2f TB/s" % (gb, gb / total,
                                                                              100 * gb / total / HBM_TBS, HBM_TBS)
                print("%-17s %10.3f (profiler, device time of %d kernels)%s" % (name, total, len(per), extra))
                for k, v in sorted(per.items(), key=lambda kv: -kv[1]):
                    print("    %8.3f ms  %s" % (v, k[:110]))
                row["kernels"][name] = entry
            results.append(row)
            del conv, x, rec, go, beta, dz, gs, gd
            torch.cuda.empty_cache()
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "nodes": n, "edges": e, "rounds": args.rounds, "results": results}, f, indent=1)
    if any(r["output_rel_err"] > (1e-4 if "float32" in r["layer"] else 3e-2) for r in results):
        raise SystemExit("bench_faconv.py: the fused output differs from the op-by-op output")


if __name__ == "__main__":
    main()
