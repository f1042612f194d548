"""Times the skip-gram negative-sampling loss on three routes, alternating within every round.

    python scripts/bench_skipgram_loss.py [--rounds 5] [--reps 10] [--out FILE]

Routes:
  - fused: pgl.nn.functional.skip_gram_loss (csrc/sgns.cu forward; csr_build + aggregation backward);
  - torch: the reference's SkipGramModel.forward restated in torch (embedding lookups, matmuls, BCEWithLogitsLoss);
  - sddmm: the op-by-op library route, pglb_sddmm_dot_f32 for the logits and the torch loss on them.  It has no
    backward, so only its forward is timed.
Workloads (batches from the device samplers on an RMAT (0.57, 0.19, 0.19, 0.05) graph of 2^20 nodes, 10^7 edges):
  - deepwalk: 512 walks of 40, window 10, 20 alias negatives, separate 2^20-node tables, D = 128, dense gradients, Adam;
  - metapath2vec: 512 two-relation metapath walks of 24, window 3, 5 in-batch negatives (cat(pos, pos[idx])), one
    shared 5e6-node table, D = 64, sparse gradients, SparseAdam;
  - all_nodes: every node walks 8 steps, window 2, 1 alias negative (about 10^7 pairs), D = 128, dense, Adam.
Before timing, the routes' losses and gradients are compared.  "forward" is timed under torch.no_grad() (the fused
kernel's loss-only form), "forward_train" with grad enabled (the fused kernel also writes c and w).  Reported per
workload and route: those two, forward + backward and full-step medians (CUDA events), peak allocated memory of one
forward + backward beyond the resident tables, and for both fused forwards the achieved bytes/s against the byte
models below and HBM3's 3.35 TB/s.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402  (graph generators)
import pgl_b200 as pgl  # noqa: E402
from pgl_b200 import ops  # noqa: E402

HBM = 3.35e12


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        name, limit = [x.strip() for x in r.stdout.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": limit}
    except Exception:
        return {"name": torch.cuda.get_device_name(0), "power_limit": "not read"}


def fwd_bytes(P, K, D):
    """The fused forward's compulsory traffic: the ids, one centre row per pair and 1 + K context rows per pair read
    (repeats counted: each use is one row read, as the kernel issues it), c and w written."""
    return 8 * P * (2 + K) + 4 * D * P * (2 + K) + 4 * P * (1 + K) + 4 * D * P


def fwd_bytes_loss_only(P, K, D):
    """The same without the c and w writes: the loss-only form under torch.no_grad()."""
    return 8 * P * (2 + K) + 4 * D * P * (2 + K)


def torch_loss(emb, ctx, src, dsts, sparse):
    src_embed = torch.nn.functional.embedding(src.reshape(-1, 1), emb, sparse=sparse)
    dsts_embed = torch.nn.functional.embedding(dsts, ctx, sparse=sparse)
    pos = torch.matmul(src_embed, dsts_embed[:, 0:1].transpose(1, 2))
    neg = torch.matmul(src_embed, dsts_embed[:, 1:].transpose(1, 2))
    bce = torch.nn.BCEWithLogitsLoss()
    return (bce(pos, torch.ones_like(pos)) + bce(neg, torch.zeros_like(neg))) / 2


def sddmm_loss(emb, ctx, src, dsts):
    P, J = dsts.shape
    D = emb.shape[1]
    s = ops.sddmm_dot(emb.detach(), ctx.detach(), src.repeat_interleave(J), dsts.reshape(-1), 1, D).reshape(P, J)
    return (torch.nn.functional.softplus(-s[:, 0]).mean() + torch.nn.functional.softplus(s[:, 1:]).mean()) / 2


ROUTES = {"fused": lambda e, c, s, d, sp: pgl.nn.functional.skip_gram_loss(e, c, s, d, sparse=sp),
          "torch": lambda e, c, s, d, sp: torch_loss(e, c, s, d, sp),
          "sddmm": lambda e, c, s, d, sp: sddmm_loss(e, c, s, d)}


def make_batches(g, hg, alias, events, n):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(3)
    starts = torch.randint(0, n, (512,), generator=gen, device="cuda")
    out = []
    walks = pgl.sampling.random_walk(g, starts, 40, seed=1)
    src, pos = pgl.sampling.skip_gram_pairs(walks, 10, seed=1)
    neg = pgl.sampling.alias_sample(alias, events, (src.numel(), 20), seed=1)
    out.append(("deepwalk", src, torch.cat([pos[:, None], neg], 1), n, 128, False, False))
    walks = pgl.sampling.metapath_randomwalk(hg, starts, "r0-r1", 24, seed=2)
    src, pos = pgl.sampling.skip_gram_pairs(walks, 3, seed=2)
    idx = torch.randint(0, pos.numel(), (pos.numel(), 5), generator=gen, device="cuda")
    out.append(("metapath2vec", src, torch.cat([pos[:, None], pos[idx]], 1), 5_000_000, 64, True, True))
    walks = pgl.sampling.random_walk(g, torch.arange(n, device="cuda"), 8, seed=3)
    src, pos = pgl.sampling.skip_gram_pairs(walks, 2, seed=3)
    neg = pgl.sampling.alias_sample(alias, events, (src.numel(), 1), seed=3)
    out.append(("all_nodes", src, torch.cat([pos[:, None], neg], 1), n, 128, False, False))
    return out


def timed(fn, reps):
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) * 1e-3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_skipgram_loss.py needs a CUDA device"
    torch.cuda.set_device(0)
    n = 1 << 20
    edges = bench.rmat_edges(torch, 20, 10_000_000, seed=1, device="cuda")
    g = pgl.Graph(edges=edges, num_nodes=n)
    half = edges.shape[0] // 2
    hg = pgl.HeterGraph(edges={"r0": edges[:half].cpu().numpy(), "r1": edges[half:].cpu().numpy()}, num_nodes=n,
                        node_types=np.zeros(n, np.int64)).tensor()
    alias, events = pgl.sampling.alias_table(g.outdegree().double() ** 0.75)
    res = {"card": card(), "workloads": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    for name, src, dsts, N, D, shared, sparse in make_batches(g, hg, alias, events, n):
        P, J = dsts.shape
        torch.manual_seed(0)
        emb = torch.nn.Parameter(torch.empty(N, D, device="cuda").uniform_(-1, 1))
        ctx = emb if shared else torch.nn.Parameter(torch.empty(N, D, device="cuda").uniform_(-0.1, 0.1))
        params = [emb] if shared else [emb, ctx]
        row = {"workload": name, "pairs": P, "negatives": J - 1, "nodes": N, "D": D, "shared": shared,
               "sparse": sparse, "routes": {}}
        # agreement before timing: losses, and the fused gradients against the torch route's
        grads = {}
        for r in ("fused", "torch"):
            for p in params:
                p.grad = None
            loss = ROUTES[r](emb, ctx, src, dsts, sparse)
            loss.backward()
            grads[r] = (float(loss), [p.grad.to_dense() if p.grad.is_sparse else p.grad for p in params])
        l_sd = float(sddmm_loss(emb, ctx, src, dsts))
        row["loss"] = {"fused": grads["fused"][0], "torch": grads["torch"][0], "sddmm": l_sd}
        assert abs(grads["fused"][0] - grads["torch"][0]) <= 1e-4 * grads["torch"][0], row["loss"]
        assert abs(l_sd - grads["torch"][0]) <= 1e-4 * grads["torch"][0], row["loss"]
        for gf, gt in zip(grads["fused"][1], grads["torch"][1]):
            err = float((gf - gt).abs().max())
            scale = float(gt.abs().max())
            row.setdefault("grad_max_abs_diff_over_max", []).append(err / scale)
            assert err <= 1e-3 * scale, (err, scale)
        del grads
        for p in params:
            p.grad = None
        opt = (torch.optim.SparseAdam if sparse else torch.optim.Adam)(params, lr=1e-3)

        def fwd(r):
            with torch.no_grad():
                ROUTES[r](emb, ctx, src, dsts, sparse)

        def fwd_train(r):
            ROUTES[r](emb, ctx, src, dsts, sparse)

        def fwdbwd(r):
            ROUTES[r](emb, ctx, src, dsts, sparse).backward()
            for p in params:
                p.grad = None

        def step(r):
            opt.zero_grad()
            ROUTES[r](emb, ctx, src, dsts, sparse).backward()
            opt.step()

        kinds = {"forward": fwd, "forward_train": fwd_train, "forward_backward": fwdbwd, "step": step}
        samples = {r: {k: [] for k in kinds} for r in ROUTES}
        for _ in range(a.rounds):
            for k, fn in kinds.items():
                for r in ROUTES:
                    if r == "sddmm" and k != "forward":
                        continue
                    samples[r][k].append(timed(lambda: fn(r), a.reps))
        for r in ROUTES:
            peak = None
            if r != "sddmm":
                for p in params:
                    p.grad = None
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                ROUTES[r](emb, ctx, src, dsts, sparse).backward()
                torch.cuda.synchronize()
                peak = torch.cuda.max_memory_allocated() - base
                for p in params:
                    p.grad = None
            row["routes"][r] = {k: float(np.median(v)) for k, v in samples[r].items() if v}
            row["routes"][r]["spread"] = {k: [float(min(v)), float(max(v))] for k, v in samples[r].items() if v}
            row["routes"][r]["peak_bytes_fwd_bwd"] = peak
        for kind, fb in (("forward", fwd_bytes_loss_only(P, J - 1, D)), ("forward_train", fwd_bytes(P, J - 1, D))):
            t = row["routes"]["fused"][kind]
            row["fused_%s_bytes" % kind] = fb
            row["fused_%s_TBps" % kind] = fb / t / 1e12
            row["fused_%s_share_of_hbm" % kind] = fb / t / HBM
        row["torch_rows_tensor_bytes"] = P * J * D * 4
        res["workloads"].append(row)
        print(json.dumps(row), flush=True)
        del emb, ctx, params, opt
        torch.cuda.empty_cache()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
