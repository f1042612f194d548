"""Where does the groups-of-8 geometry of spmm_v5_kernel start to win?  Chung-Lu graphs (exponent 0.8, permuted ids) of
2M nodes and 16 / 24 / 32 / 40 slots per row, 128-float rows, sum; run once with PGLB_V5_GEO=0 (groups of 4) and once
with PGLB_V5_GEO=2 (groups of 8); the library reads it once per process."""
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

dev = torch.device("cuda", 0)
torch.cuda.set_device(dev)
n = int(os.environ.get("GEO_SWEEP_NODES", "2000000"))
x = bench.gen_features(torch, n, 128, 9, dev)
for deg in [int(v) for v in os.environ.get("GEO_SWEEP_DEGS", "16,24,32,40").split(",")]:
    edges = bench.gen_edges(torch, n, n * deg, 0.8, 31 + deg, dev)
    g = pgl.Graph(edges=edges, num_nodes=n)
    fwd = g._fwd_csr()
    packed = ops._packed_of(fwd, x)
    out = torch.empty(n, 128, device=dev)

    def step():
        return ops._spmm_raw(fwd["indptr"], fwd["cols"], x, n, "sum", max_degree=fwd["max_degree"], out=out, packed=packed)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    per = []
    for _ in range(10):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        step()
        b.record()
        torch.cuda.synchronize()
        per.append(a.elapsed_time(b))
    print(json.dumps({"nodes": n, "slots_per_row": deg, "geo_env": os.environ.get("PGLB_V5_GEO", "auto"), "ms_mean": float(np.mean(per)),
                      "ms_min": float(np.min(per)), "G_edges_s": n * deg / np.mean(per) / 1e6}), flush=True)
    del g, fwd, packed, edges
    torch.cuda.empty_cache()
