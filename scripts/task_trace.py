"""Per-task timeline of the fused GAT aggregation on cfg3 (pglb_debug_task_trace): where the launch's time goes by task
id, how many warps are busy over time, the longest tasks.  One JSON line."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import pgl_b200 as pgl  # noqa: E402
from pgl_b200 import ops  # noqa: E402
from pgl_b200._lib import check, lib  # noqa: E402


def analyse(tr, label, extra):
    tr = tr[tr[:, 1] > 0]
    nt = len(tr)
    t0 = tr[:, 0].min()
    st, en = (tr[:, 0] - t0) / 1e3, (tr[:, 1] - t0) / 1e3        # microseconds
    dur = en - st
    span = en.max()
    nb = 20
    edges_t = np.linspace(0, span, nb + 1)
    busy = []
    for i in range(nb):
        lo, hi = edges_t[i], edges_t[i + 1]
        ov = np.clip(np.minimum(en, hi) - np.maximum(st, lo), 0, None).sum() / (hi - lo)
        busy.append(round(float(ov), 1))
    dec = [round(float(dur[i * nt // 10:(i + 1) * nt // 10].mean()), 1) for i in range(10)]
    top = np.argsort(-dur)[:8]
    out = {"case": label, "tasks": int(nt), "span_us": round(float(span), 1), "sum_task_us": round(float(dur.sum()), 0),
           "dur_us_p50_p90_p99_max": [round(float(np.percentile(dur, q)), 1) for q in (50, 90, 99, 100)],
           "mean_dur_us_by_task_id_decile": dec, "busy_warps_by_time_bucket": busy,
           "last_start_us": round(float(st.max()), 1),
           "longest": [[int(i), round(float(dur[i]), 1), round(float(st[i]), 1)] for i in top], "sms_used": int(len(np.unique(tr[:, 2])))}
    out.update(extra)
    print(json.dumps(out), flush=True)


def main():
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    n, e, H, Dh = 1 << 20, 10_000_000, 8, 16
    edges = bench.rmat_edges(torch, 20, e, seed=1, device=dev)
    g = pgl.Graph(edges=edges, num_nodes=n)
    x = bench.gen_features(torch, n, 128, 2, dev)
    torch.manual_seed(3)
    conv = pgl.nn.GATConv(128, Dh, feat_drop=0, attn_drop=0, num_heads=H).to(dev).eval()
    csr = g._fwd_csr()
    cap = 1 << 20
    buf = torch.zeros(cap, 4, dtype=torch.int64, device=dev)
    with torch.no_grad():
        f = (x @ conv.linear.weight + conv.linear.bias).reshape(-1, H, Dh).contiguous()
        a_s = (f * conv.weight_src).sum(-1).contiguous()
        a_d = (f * conv.weight_dst).sum(-1).contiguous()
        for _ in range(3):
            ops.gat_fused(csr, f, a_s, a_d, 0.2)
        torch.cuda.synchronize()
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(10):
            ops.gat_fused(csr, f, a_s, a_d, 0.2)
        ev1.record()
        torch.cuda.synchronize()
        ms = ev0.elapsed_time(ev1) / 10
        buf.zero_()
        check(lib.pglb_debug_task_trace(ops._ptr(buf), cap))
        ops.gat_fused(csr, f, a_s, a_d, 0.2)
        torch.cuda.synchronize()
        check(lib.pglb_debug_task_trace(None, 0))
        analyse(buf.cpu().numpy(), "cfg3 fused GAT", {"ms_untraced": round(ms, 3),
                                                      "task_env": os.environ.get("PGLB_STREAM_TASK", "default")})


if __name__ == "__main__":
    main()
