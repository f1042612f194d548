"""Graph-level readouts on one GPU: the fused attention readout (gate = GlobalAttention, query = Set2Set) against a
torch restatement of the reference's op order (pgl/nn/pool.py:139-142, 173-178: score, 7-op segment softmax,
multiply, segment_sum), forward and forward + backward; segment top-k on both of its paths; pad / unpad bandwidth.

    python scripts/bench_readout.py [--reps 10] [--workloads mol,infer,large]

Prints one JSON line per workload.  Times are medians of CUDA-event intervals over --reps calls after two warm-up
calls.  GB/s are algorithmic bytes over kernel time, reported beside the 3.35 TB/s data-sheet bandwidth of the H100
SXM; bytes per call:
  forward : N*D*4 (x) + N*4 (gate) or B*D*4 (query) + B*D*4 (out) + B*4 (lse) + (B+1)*8 (indptr)
  backward: N*D*4 (x) + N*4 (gate) or B*D*4 (query) + 2*B*D*4 (out, grad_out) + B*4 (lse) + (B+1)*8 (indptr)
            + N*D*4 (grad_x) + N*4 (grad_gate) or B*D*4 (grad_query)
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

PEAK_TBS = 3.35


def card():
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout
        power = float(out.strip().splitlines()[0])
    except Exception:
        power = None
    return name, power


def timed(fn, reps):
    for _ in range(2):
        fn()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def kernels_of(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def torch_readout(x, ids, B, gate=None, query=None):
    s = (x * query[ids]).sum(-1) if gate is None else gate
    m = torch.full((B,), -torch.inf, device=x.device).scatter_reduce(0, ids, s, "amax")
    e = torch.exp(s - m[ids])
    den = torch.zeros(B, device=x.device).index_add(0, ids, e)
    a = (e / den[ids]).unsqueeze(1)
    return torch.zeros(B, x.shape[1], device=x.device).index_add(0, ids, a * x)


def workload(name):
    rng = np.random.default_rng(0)
    if name == "mol":
        return rng.integers(10, 41, 256), 300
    if name == "infer":
        return rng.integers(20, 33, 65536), 300
    if name == "large":
        return np.full(8, 1_000_000), 128
    raise ValueError(name)


def run(name, reps, pgl):
    sizes, D = workload(name)
    B, N = len(sizes), int(sizes.sum())
    dev = torch.device("cuda")
    ip = torch.as_tensor(np.concatenate([[0], np.cumsum(sizes)]), dtype=torch.int64, device=dev)
    ids = torch.repeat_interleave(torch.arange(B, device=dev), ip[1:] - ip[:-1])
    x = torch.randn(N, D, device=dev)
    gate = torch.randn(N, device=dev)
    query = torch.randn(B, D, device=dev) / D ** 0.5
    gout = torch.randn(B, D, device=dev)
    pgl.ops.segment_max_len(ip)
    res = {"workload": name, "B": B, "N": N, "D": D, "max_len": int(sizes.max())}
    for mode in ("gate", "query"):
        kw = {"gate": gate} if mode == "gate" else {"query": query}
        fwd_bytes = N * D * 4 + (N * 4 if mode == "gate" else B * D * 4) + B * D * 4 + B * 4 + (B + 1) * 8
        bwd_bytes = N * D * 4 + (N * 4 if mode == "gate" else B * D * 4) + 2 * B * D * 4 + B * 4 + (B + 1) * 8 + \
            N * D * 4 + (N * 4 if mode == "gate" else B * D * 4)

        def fused_fwd():
            with torch.no_grad():
                pgl.ops.attn_readout(x, ip, **kw)

        def torch_fwd():
            with torch.no_grad():
                torch_readout(x, ids, B, **kw)

        xg = x.clone().requires_grad_(True)
        kg = {k: v.clone().requires_grad_(True) for k, v in kw.items()}

        def fused_train():
            (pgl.ops.attn_readout(xg, ip, **kg) * gout).sum().backward()

        def torch_train():
            (torch_readout(xg, ids, B, **kg) * gout).sum().backward()

        l0 = pgl.ops.launch_count()
        fused_fwd()
        torch.cuda.synchronize()
        launches = pgl.ops.launch_count() - l0
        t_f = timed(fused_fwd, reps)
        t_t = timed(torch_fwd, reps)
        t_ft = timed(fused_train, reps)
        t_tt = timed(torch_train, reps)
        # backward kernel alone: forward + backward minus forward, from the same medians
        t_b = max(t_ft - t_f, 1e-6)
        res[mode] = {
            "fused_fwd_ms": round(t_f, 4), "torch_fwd_ms": round(t_t, 4),
            "fused_fwd_bwd_ms": round(t_ft, 4), "torch_fwd_bwd_ms": round(t_tt, 4),
            "fused_fwd_launches": launches, "torch_fwd_kernels": kernels_of(torch_fwd),
            "fwd_GBps": round(fwd_bytes / t_f / 1e6, 1), "fwd_of_peak": round(fwd_bytes / t_f / 1e9 / PEAK_TBS, 3),
            "bwd_GBps_est": round(bwd_bytes / t_b / 1e6, 1),
        }
    # the layer path: GlobalAttention / Set2Set(2 iterations) on a batched Graph.  "first call" includes reading the
    # batch's segment CSR off the graph (one read back); later calls reuse it.
    graph = pgl.Graph(num_nodes=N, edges=torch.zeros((0, 2), dtype=torch.int64, device=dev), _graph_node_index=ip,
                      _num_graph=B)
    ga = pgl.nn.GlobalAttention(pgl.nn.Linear(D, 1)).to(dev)
    s2s = pgl.nn.Set2Set(D, 2).to(dev)

    def layer(mod, cold):
        def fn():
            if cold:
                graph.__dict__.pop("_pglb_readout_csr", None)
            with torch.no_grad():
                mod(graph, x)
        return fn
    res["layer"] = {"global_attention_ms": round(timed(layer(ga, False), reps), 4),
                    "global_attention_first_call_ms": round(timed(layer(ga, True), reps), 4),
                    "set2set_2iter_ms": round(timed(layer(s2s, False), reps), 4),
                    "set2set_2iter_first_call_ms": round(timed(layer(s2s, True), reps), 4)}
    scores = torch.randn(N, device=dev)

    def topk():
        pgl.ops.segment_topk_perm(scores, ip, 0.5)
    res["topk"] = {"path": "smem" if int(sizes.max()) <= 2048 else "radix_sort", "ms": round(timed(topk, reps), 4)}
    L = int(sizes.max())
    pad_bytes = N * D * 4 + B * L * D * 4
    t_pad = timed(lambda: pgl.ops.segment_pad(x, ip, L), reps)
    padded = pgl.ops.segment_pad(x, ip, L)
    t_unpad = timed(lambda: pgl.ops.segment_unpad(padded, ip, N), reps)
    res["pad"] = {"ms": round(t_pad, 4), "GBps": round(pad_bytes / t_pad / 1e6, 1)}
    res["unpad"] = {"ms": round(t_unpad, 4), "GBps": round(2 * N * D * 4 / t_unpad / 1e6, 1)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--workloads", default="mol,infer,large")
    args = ap.parse_args()
    import pgl_b200 as pgl
    torch.cuda.set_device(0)
    name, power = card()
    for w in args.workloads.split(","):
        r = run(w, args.reps, pgl)
        r.update({"gpu": name, "power_limit_w": power})
        print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
