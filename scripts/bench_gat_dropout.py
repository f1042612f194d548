"""GATConv training with attention dropout on cfg3: the fused kernels against the op-by-op route.

Builds bench_gat.py's cfg3 graph (RMAT scale 20, 10M edges) and GATConv(128 -> 8 heads x 16, feat_drop = 0), then,
for float32 and bfloat16 modules, times forward + backward of three variants that alternate inside every round:
  * fused_drop:    attn_drop = 0.6 on the fused kernels (the *_drop_* entries);
  * op_by_op_drop: attn_drop = 0.6 with ops.GAT_FUSED_TRAIN = False (send_uv + LeakyReLU + edge_softmax + nn.Dropout
                   + send_ue_recv: the route every GATConv with attention dropout took before);
  * fused_nodrop:  attn_drop = 0 on the fused kernels.
It also times the two kernels that gained the in-kernel Philox stream on their own (the training forward aggregation
and the edge backward, float32, with and without dropout), so the stream's cost is visible apart from the layer.
Checks, at full size: the float32 fused dropout output against plain torch with the same mask (relative error
<= 1e-4 of the largest output), and the bfloat16 one bit for bit against the float32 dropout kernel on the widened
features, rounded.

    python scripts/bench_gat_dropout.py [--rounds 5] [--layer-steps 5] [--steps 20] [--json FILE]
"""
import argparse
import ctypes
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
from pgl_b200 import _lib, ops  # noqa: E402

P_DROP = 0.6
SEED = (20261016, 0)


def edge_mask(csr, H, p, seed):
    """[E, H] float32 keep mask in edge order (the library's host restatement of the kernels' stream)."""
    E = int(csr["cols"].shape[0])
    w = np.zeros(E, np.uint32)
    _lib.check(_lib.lib.pglb_attn_dropout_keep_host(seed[0], seed[1], p, 0, E, H, w.ctypes.data_as(ctypes.c_void_p)))
    bits = ((w[:, None] >> np.arange(H, dtype=np.uint32)) & 1).astype(np.float32)
    m = np.empty_like(bits)
    eid = csr.get("eid")
    m[np.arange(E) if eid is None else eid.cpu().numpy()] = bits
    return torch.from_numpy(m).cuda()


def torch_drop_ref(f, a_s, a_d, src, dst, n, slope, mask, s):
    """sum_j s m_j softmax_j(leaky(a_s[src_j] + a_d[d])) f[src_j] in plain torch fp32."""
    z = torch.nn.functional.leaky_relu(a_s[src] + a_d[dst], slope)
    H = z.shape[1]
    m = torch.full((n, H), -float("inf"), device=z.device).scatter_reduce(0, dst[:, None].expand(-1, H), z, "amax")
    pe = torch.exp(z - m[dst])
    beta = pe / torch.zeros((n, H), device=z.device).index_add(0, dst, pe)[dst] * mask * s
    del z, pe
    out = torch.zeros_like(f)
    for c0 in range(0, int(src.shape[0]), 1 << 22):   # chunks: f[src] of 10M edges is 5 GB
        sl = slice(c0, c0 + (1 << 22))
        out.index_add_(0, dst[sl], f[src[sl]] * beta[sl].unsqueeze(-1))
    return out


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
        raise SystemExit("bench_gat_dropout.py: no CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = gpu_info()
    n, e, H, Dh = 1 << args.scale, args.edges, 8, 16
    D = H * Dh
    edges = rmat(args.scale, e)
    g = pgl.Graph(edges=edges, num_nodes=n)
    fwd = g._fwd_csr()
    bwd = g._bwd_csr()
    E = int(fwd["cols"].shape[0])
    torch.manual_seed(2)
    x = torch.randn(n, 128, device=dev)
    conv = pgl.nn.GATConv(128, Dh, feat_drop=0, attn_drop=P_DROP, num_heads=H).to(dev)
    with torch.no_grad():
        f32 = (x @ conv.linear.weight + conv.linear.bias).reshape(-1, H, Dh).contiguous()
        a_s = (f32 * conv.weight_src).sum(-1).contiguous()
        a_d = (f32 * conv.weight_dst).sum(-1).contiguous()
    s32 = float(np.float32(1.0 / (1.0 - float(np.float32(P_DROP)))))

    # 1. checks at full size
    with torch.no_grad():
        got = ops.gat_fused_train(fwd, bwd, f32, a_s, a_d, 0.2, attn_drop=P_DROP, seed=SEED)
        src, dst = edges[:, 0].contiguous(), edges[:, 1].contiguous()   # edge order = edge ids
        ref = torch_drop_ref(f32, a_s, a_d, src, dst, n, 0.2, edge_mask(fwd, H, P_DROP, SEED), s32)
        rel = float((got - ref).abs().max() / ref.abs().max())
        del ref, src, dst
        got16 = ops.gat_fused_train(fwd, bwd, f32.to(torch.bfloat16), a_s, a_d, 0.2, out_dtype=torch.bfloat16,
                                    attn_drop=P_DROP, seed=SEED)
        ref16 = ops.gat_fused_train(fwd, bwd, f32.to(torch.bfloat16).float(), a_s, a_d, 0.2, attn_drop=P_DROP,
                                    seed=SEED).to(torch.bfloat16)
        bf16_bits = bool(torch.equal(got16.view(torch.int16), ref16.view(torch.int16)))
        del got, got16, ref16
    torch.cuda.empty_cache()

    # 2. the two kernels with the Philox stream, alone (float32 entries, alternating with and without dropout)
    f2 = f32.reshape(n, D)
    out = torch.empty((n, D), device=dev)
    lse = torch.zeros((n, H), device=dev)
    go = torch.randn(n, D, device=dev)
    alpha = torch.empty((E, H), device=dev)
    dz = torch.empty((E, H), device=dev)
    need = ctypes.c_size_t(0)
    _lib.check(_lib.lib.pglb_spmm_csr_ws(n, E, D, ctypes.byref(need)))
    ws = ops.workspace(dev, need.value)
    P = ops._ptr

    def k_fwd(drop):
        a = (P(fwd["indptr"]), P(fwd["cols"]), P(f2), D, P(a_s), P(a_d), 0.2, P(out), D, P(lse), n, n, E, H, Dh)
        if drop:
            _lib.check(_lib.lib.pglb_gat_fused_train_drop_csr_f32(*a, P_DROP, *SEED, P(ws), ws.numel(), ops._stream()))
        else:
            _lib.check(_lib.lib.pglb_gat_fused_train_csr_f32(*a, P(ws), ws.numel(), ops._stream()))

    def k_bwd(drop):
        a = (P(fwd["rows"]), P(fwd["cols"]), P(fwd["eid"]), P(f2), D, P(go), D, P(out), D, P(a_s), P(a_d), P(lse), 0.2,
             E, H, Dh)
        if drop:
            _lib.check(_lib.lib.pglb_gat_bwd_edge_drop_f32(*a, P_DROP, *SEED, P(alpha), P(dz), ops._stream()))
        else:
            _lib.check(_lib.lib.pglb_gat_bwd_edge_f32(*a, P(alpha), P(dz), ops._stream()))

    kernels = {("forward", False): lambda: k_fwd(False), ("forward", True): lambda: k_fwd(True),
               ("edge_backward", False): lambda: k_bwd(False), ("edge_backward", True): lambda: k_bwd(True)}
    ktimes = {k: [] for k in kernels}
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
    for rnd in range(args.rounds):
        keys = list(kernels)
        for k in (keys if rnd % 2 == 0 else keys[::-1]):
            kernels[k]()   # warm-up (and the forward's lse for the backward)
            torch.cuda.synchronize()
            for a, b in evs:
                a.record()
                kernels[k]()
                b.record()
            torch.cuda.synchronize()
            ktimes[k] += [a.elapsed_time(b) for a, b in evs]
    del out, lse, go, alpha, dz, f2
    torch.cuda.empty_cache()

    # 3. GATConv forward + backward
    variants = (("fused_drop", P_DROP, True), ("op_by_op_drop", P_DROP, False), ("fused_nodrop", 0.0, True))
    results = {}
    for dname, dt in (("fp32", torch.float32), ("bf16", torch.bfloat16)):
        mods = {}
        for name, p, fused in variants:
            m = pgl.nn.GATConv(128, Dh, feat_drop=0, attn_drop=p, num_heads=H).to(dev)
            m.load_state_dict(conv.state_dict())
            mods[name] = (m.to(dt).train(), fused)
        times = {k: [] for k in mods}
        faster = []
        for rnd in range(args.rounds):
            names = list(mods)
            order = names[rnd % len(names):] + names[:rnd % len(names)]
            med = {}
            for name in order:
                m, fused = mods[name]
                xin = x.to(dt).requires_grad_()

                def fb():
                    o = m(g, xin)
                    o.float().sum().backward()
                    xin.grad = None
                    m.zero_grad(set_to_none=True)
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
                times[name] += t
                med[name] = float(np.median(t))
            faster.append(med["fused_drop"] < med["op_by_op_drop"])
        results[dname] = (times, faster)
        del mods
        torch.cuda.empty_cache()

    print("# %s | cfg3 RMAT scale %d, %d edges, GATConv(128 -> %d x %d), attn_drop %.1f | %d rounds, variants "
          "alternate in each round" % (info, args.scale, e, H, Dh, P_DROP, args.rounds))
    print("# full-size check: fp32 fused dropout vs torch with the same mask: max rel err %.2e (bar 1e-4); bf16 vs the "
          "rounded fp32 dropout kernel: %s" % (rel, "identical" if bf16_bits else "DIFFERENT"))
    print("%34s %9s %9s %9s" % ("kernel (fp32)", "median_ms", "p10_ms", "p90_ms"))
    krows = {}
    for (kname, drop), t in ktimes.items():
        med, p10, p90 = stats(t)
        label = "%s %s" % (kname, "attn_drop 0.6" if drop else "no dropout")
        krows[label] = {"median_ms": med, "p10_ms": p10, "p90_ms": p90}
        print("%34s %9.3f %9.3f %9.3f" % (label, med, p10, p90))
    print("%34s %9s %9s %9s %22s" % ("GATConv fwd+bwd", "median_ms", "p10_ms", "p90_ms", "fused_drop faster"))
    lrows = {}
    for dname, (times, faster) in results.items():
        for name, t in times.items():
            med, p10, p90 = stats(t)
            label = "%s %s" % (dname, name)
            fs = "%d/%d rounds" % (sum(faster), len(faster)) if name == "fused_drop" else ""
            lrows[label] = {"median_ms": med, "p10_ms": p10, "p90_ms": p90}
            print("%34s %9.3f %9.3f %9.3f %22s" % (label, med, p10, p90, fs))
        lrows[dname + " fused_drop_faster_than_op_by_op_in_rounds"] = faster
    if args.json:
        with open(args.json, "w") as fh:
            json.dump({"gpu": info, "nodes": n, "edges": e, "heads": H, "head_dim": Dh, "attn_drop": P_DROP,
                       "rounds": args.rounds, "max_rel_err_fp32": rel, "bf16_bit_identical": bf16_bits,
                       "kernels": krows, "gatconv_fwd_bwd": lrows}, fh, indent=1)
    if rel > 1e-4 or not bf16_bits:
        raise SystemExit("bench_gat_dropout.py: the fused dropout output fails its check")


if __name__ == "__main__":
    main()
