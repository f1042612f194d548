"""The fused K-hop propagation step (ops.propagate) against the op-by-op hop it replaces, alternating in every round.

For each case below, both routes run the same layer; the op-by-op route is the layer with ops.propagate declining
every call (its fallback is the parent's code).  Before timing, the fused output is compared with the op-by-op one on
the full graph (bit for bit).  Times are CUDA-event medians over the rounds; the card name, power limit and max SM
clock are read (nvidia-smi, read-only) in the same run.
  * APPNP(k = 10, alpha = 0.1): inference, and a training step with a Linear in front, on cfg5's graph (bench.py's
    Chung-Lu generator, 10M nodes / 100M edges) at D = 128 (wide-row route) and D = 64 (narrow route), and on cfg4's
    products-shape graph (2.45M nodes / 124M edges) at D = 47 (node-parallel route);
  * SSGCConv(k = 16) smoothing and a GPRConv(k = 10, PPR) training step at the same shapes (inference at cfg5's
    D = 128, where the training step, which keeps every hop's output for temp's gradient, does not fit 80 GB on
    either route);
  * the reference citation_benchmark APPNP (D = 7), GCNII (k = 64, D = 64) and SSGC (k = 16 over the raw 1433-d
    features) models on Cora: a training step, and SSGC's smoothing;
  * the peak memory of one training step on either route.

Byte model of one hop, [N, D] fp32 = 4 N D bytes (P below), aggregation A = E (4 D + 8) + P + 8 N + 8 N:
    op-by-op APPNP / GCNII: A + 3 elementwise passes (alpha * h0, (1 - alpha) * f, the sum) = A + 7 P
    fused APPNP / GCNII:    A + P (h0)
    op-by-op SSGC:          A + 2 passes (scale, running sum) = A + 5 P;  fused: A + 2 P (acc in, acc out)
    op-by-op GPR:           A + 2 passes (temp * f, running sum) = A + 5 P;  fused: A + 2 P

    python scripts/bench_propagate.py [--rounds 5] [--skip-big] [--json FILE]
"""
import argparse
import contextlib
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)
import bench  # noqa: E402
import pgl_b200 as pgl  # noqa: E402
from bench_half import gpu_info, stats  # noqa: E402
from oracle import oracle as O  # noqa: E402
from pgl_b200 import ops  # noqa: E402
from pgl_b200.nn import conv as C  # noqa: E402


@contextlib.contextmanager
def op_by_op():
    """every ops.propagate call declines: the layers run their op-by-op hop"""
    real = ops.propagate
    ops.propagate = lambda *a, **k: None
    try:
        yield
    finally:
        ops.propagate = real


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def peak_gb(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return (torch.cuda.max_memory_allocated() - base) / 1e9


def compare(name, fn, rounds, results, bytes_model=None, memory=False):
    """fn() -> output tensor; runs once per route for the check and the warm-up, then `rounds` alternating pairs"""
    a = fn()
    with op_by_op():
        b = fn()
    identical = bool(torch.equal(a, b))
    del a, b
    tf, to = [], []
    for _ in range(rounds):
        tf.append(timed(fn))
        with op_by_op():
            to.append(timed(fn))
    row = {"case": name, "fused_ms": stats(tf), "op_by_op_ms": stats(to), "bit_identical": identical,
           "fused_faster_rounds": "%d/%d" % (sum(f < o for f, o in zip(tf, to)), rounds),
           "speedup": stats(to)[0] / stats(tf)[0]}
    if bytes_model:
        row["model_gb_fused"], row["model_gb_op"] = bytes_model
    if memory:
        row["peak_gb_fused"] = peak_gb(fn)
        with op_by_op():
            row["peak_gb_op"] = peak_gb(fn)
    results.append(row)
    print("%-44s fused %9.3f ms  op-by-op %9.3f ms  x%.3f  faster %s  %s%s" % (
        name, row["fused_ms"][0], row["op_by_op_ms"][0], row["speedup"], row["fused_faster_rounds"],
        "identical" if identical else "DIFFERENT",
        ("  peak GB %.2f / %.2f" % (row["peak_gb_fused"], row["peak_gb_op"])) if memory else ""), flush=True)


def hop_gb(n, e, d, extra_passes):
    p = 4.0 * n * d
    return (e * (4 * d + 8) + p + 16 * n + extra_passes * p) / 1e9


def big_cases(name, g, n, e, d, rounds, results, k_appnp=10):
    torch.manual_seed(1)
    x = bench.gen_features(torch, n, d, 3, "cuda")
    appnp = C.APPNP(alpha=0.1, k_hop=k_appnp)
    lin = C.Linear(d, d).cuda()

    def appnp_inf():
        with torch.no_grad():
            return appnp(g, x)

    def appnp_train():
        lin.zero_grad(set_to_none=True)
        out = appnp(g, lin(x))
        out.square().mean().backward()
        return out.detach()

    ssgc = C.SSGCConv(d, 16, k_hop=16, cached=False).cuda()

    def ssgc_smooth():
        with torch.no_grad():
            return ssgc._smooth(g, x)

    gpr = C.GPRConv(d, d, d, drop=0.0, dprate=0.0, k_hop=10).cuda()

    def gpr_train():
        gpr.zero_grad(set_to_none=True)
        out = gpr(g, x)
        out.square().mean().backward()
        return out.detach()

    def gpr_inf():
        with torch.no_grad():
            return gpr(g, x)

    compare("%s APPNP k=10 inference D=%d" % (name, d), appnp_inf, rounds, results,
            (k_appnp * hop_gb(n, e, d, 1), k_appnp * hop_gb(n, e, d, 7)))
    compare("%s APPNP k=10 train step D=%d" % (name, d), appnp_train, rounds, results, memory=True)
    compare("%s SSGC k=16 smoothing D=%d" % (name, d), ssgc_smooth, rounds, results,
            (16 * hop_gb(n, e, d, 2), 16 * hop_gb(n, e, d, 5)))
    if 4.0 * n * d * 15 < 60e9:
        compare("%s GPR k=10 train step D=%d" % (name, d), gpr_train, rounds, results, memory=True)
    else:
        # both routes keep every hop's output for temp's gradient: 10 x 5.1 GB at cfg5, D = 128, which with the MLP's
        # activations does not fit 80 GB on either route
        compare("%s GPR k=10 inference D=%d" % (name, d), gpr_inf, rounds, results)
    del x


class CoraAPPNP(torch.nn.Module):
    def __init__(self, din, ncls, hidden=64):
        super().__init__()
        self.l1, self.l2 = C.Linear(din, hidden), C.Linear(hidden, ncls)
        self.drop = torch.nn.Dropout(0.5)
        self.prop = C.APPNP(alpha=0.1, k_hop=10)

    def forward(self, g, x):
        return self.prop(g, self.l2(self.drop(torch.relu(self.l1(self.drop(x))))))


class CoraGCNII(torch.nn.Module):
    def __init__(self, din, ncls, hidden=64, k=64):
        super().__init__()
        self.l1, self.l2 = C.Linear(din, hidden), C.Linear(hidden, ncls)
        self.drop = torch.nn.Dropout(0.6)
        self.conv = C.GCNII(hidden, activation="relu", lambda_l=0.5, alpha=0.1, k_hop=k, dropout=0.6)

    def forward(self, g, x):
        h = torch.relu(self.l1(self.drop(x)))
        return self.l2(self.drop(self.conv(g, h)))


def cora_cases(rounds, results):
    cora = O.load_cora(os.path.join(ROOT, "tests", "golden", "cora.npz"))
    n = cora["num_nodes"]
    g = pgl.Graph(edges=cora["edges"], num_nodes=n)
    g.tensor()
    x = torch.from_numpy(cora["x"]).cuda()
    y = torch.from_numpy(cora["y"]).cuda()
    tr = torch.from_numpy(cora["train_index"]).cuda()
    ncls = cora["num_classes"]
    for name, model in (("Cora APPNP (D=7) train step", CoraAPPNP(1433, ncls)),
                        ("Cora GCNII k=64 (D=64) train step", CoraGCNII(1433, ncls))):
        model = model.cuda().eval()   # dropout off: the routes' outputs are compared bit for bit
        opt = torch.optim.Adam(model.parameters(), lr=0.01)

        def step(model=model, opt=opt):
            out = model(g, x)
            loss = torch.nn.functional.cross_entropy(out[tr], y[tr])
            opt.zero_grad()
            loss.backward()
            return out.detach()
        compare(name, step, rounds * 4, results, memory=True)
    ssgc = C.SSGCConv(1433, ncls, k_hop=16, cached=False).cuda()

    def smooth():
        with torch.no_grad():
            return ssgc._smooth(g, x)

    def ssgc_step():
        out = ssgc(g, x)
        torch.nn.functional.cross_entropy(out[tr], y[tr]).backward()
        return out.detach()
    compare("Cora SSGC k=16 smoothing (D=1433)", smooth, rounds * 4, results)
    compare("Cora SSGC k=16 train step (D=1433)", ssgc_step, rounds * 4, results)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-big", action="store_true", help="Cora only")
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    info = gpu_info()
    print("GPU (name, power limit, max SM clock):", info)
    results = []
    cora_cases(args.rounds, results)
    if not args.skip_big:
        n, e = 10_000_000, 100_000_000
        edges = bench.gen_edges(torch, n, e, 0.8, 20240922, "cuda")
        g = pgl.Graph(edges=edges, num_nodes=n)
        g.tensor()
        del edges
        for d in (128, 64):
            big_cases("cfg5", g, n, e, d, args.rounds, results)
        del g
        torch.cuda.empty_cache()
        n4, und = 2_449_029, 61_859_140
        half = bench.gen_edges(torch, n4, und, 0.6, 5, "cuda")
        edges = torch.cat([half, half.flip(1)], 0)
        del half
        g4 = pgl.Graph(edges=edges, num_nodes=n4)
        g4.tensor()
        big_cases("cfg4", g4, n4, int(edges.shape[0]), 47, args.rounds, results)
    if args.json:
        with open(args.json, "w") as f:
            json.dump({"gpu": info, "rounds": args.rounds, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
