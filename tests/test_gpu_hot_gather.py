"""Hot rows of the wide-row aggregation (spmm_v5_kernel with L2 hints, D = 128): a row whose packed id has bit 31 set
is gathered by per-lane cp.async (LDGSTS), every other row by a bulk copy.  The output must be bit for bit what the
kernel gives with no hints (every row by bulk copy) and with every row hot (every row by per-lane LDGSTS): for groups
that are all cold, mixed and all hot, in both ring geometries, with streamed and gathered source norms, for the
unscaled sum and the mean, with hub rows cut into task partials and with empty rows."""
import hashlib
import json
import os
import subprocess
import sys

import pytest
import torch

from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
EMPTY = 100  # trailing nodes without any edge: empty rows and never-gathered sources


def _packings(ops, cols, n_src):
    """name -> (packed ids, has_hints).  pack_cols gives no hints once the budget covers every source, so the
    every-row-hot ids are built directly."""
    packs = {name: tuple(ops.pack_cols(cols, n_src, 512, budget_bytes=b))
             for name, b in (("none", 0), ("few", 8 * 512), ("mixed", 1 << 20))}
    assert not packs["none"][1] and packs["few"][1] and packs["mixed"][1]
    packs["all"] = (cols.to(torch.int32) | -(1 << 31), True)
    return packs


def _digests():
    """case -> {packing: sha256 of the output}, every case the kernel takes with 512-byte rows."""
    import pgl_b200 as pgl
    import pgl_b200.nn.functional as GF
    from pgl_b200 import ops
    res = {}
    for avg_deg in (5, 15):              # v5_geo: groups of 4 below 12 slots per row, groups of 8 above
        n = 20000
        edges = O.chung_lu_edges(n, n * avg_deg, exponent=0.8, seed=avg_deg)
        N = n + EMPTY
        g = pgl.Graph(edges=edges, num_nodes=N)
        g.tensor()
        fwd = g._fwd_csr()
        norm = GF.degree_norm(g).reshape(-1)
        assert fwd["slot_scale"](norm) is None and fwd["slot_scale"](norm) is not None
        x = torch.randn(N, 128, device="cuda", generator=torch.Generator("cuda").manual_seed(avg_deg))
        packs = _packings(ops, fwd["cols"], N)

        def run(case, pk):
            kw = dict(max_degree=fwd["max_degree"], packed=pk)
            if case.startswith("gcn"):
                kw.update(scale_src=norm, scale_dst=norm)
                if case == "gcn_streamed":
                    kw["packed"] = ops.PackedCols(pk, fwd["slot_scale"])
            out = ops._spmm_raw(fwd["indptr"], fwd["cols"], x, N, "mean" if case == "mean" else "sum", **kw)
            return hashlib.sha256(out.cpu().numpy().tobytes()).hexdigest()

        for case in ("gcn_gathered", "gcn_streamed", "sum", "mean"):
            res["deg%d/%s" % (avg_deg, case)] = {name: run(case, pk) for name, pk in packs.items()}
    return res


def _mismatches(digests):
    return {case: d for case, d in digests.items() if len(set(d.values())) != 1}


def _child(env):
    code = ("import sys, json; sys.path[:0] = [%r, %r]; import test_gpu_hot_gather as t; "
            "print(json.dumps(t._digests()))" % (ROOT, HERE))
    r = subprocess.run([sys.executable, "-s", "-c", code], env=dict(os.environ, **env), capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


@pytest.mark.gpu
def test_hot_rows_bit_identical_to_bulk_and_ldgsts_ring():
    """Every packing agrees with the no-hint (all bulk copy) output, the every-row-hot packing (all per-lane LDGSTS)
    included."""
    assert _mismatches(_digests()) == {}


@pytest.mark.gpu
def test_hot_rows_bit_identical_with_short_tasks():
    """Tasks of 64 slots cut every hub row into partials added by the fix-up kernel: the hybrid gather agrees with
    the no-hint and the every-row-hot outputs at that task size."""
    assert _mismatches(_child({"PGLB_STREAM_TASK": "64"})) == {}
