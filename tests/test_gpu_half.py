"""bfloat16 / float16 features on the send/recv path (pglb_spmm_csr_x16 and the widen-through ops).

Contract: messages are widened to fp32 exactly, reduced in fp32 in the fp32 kernels' slot order, and every output is
rounded once.  So a 16-bit output equals round16(the fp32 reduction) bit for bit wherever both take the same kernel
(the sequential oracle for rows of <= 1024 slots, the fp32 library on the wide-row path), and meets
|out - ref32| <= 2 u |ref32| (u = 2^-8 bf16, 2^-11 fp16) everywhere else."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DTYPES = (torch.bfloat16, torch.float16)
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
EMPTY = 100  # trailing nodes without an edge: empty rows


def _bits(t):
    return t.contiguous().view(torch.int16)


def _within_bar(out, ref32, dtype):
    out = out.double().cpu()
    ref = torch.as_tensor(ref32).double().cpu()
    return float((out - ref).abs().max()) <= 2 * U[dtype] * float(ref.abs().max())


def _graph(pgl, n, e, seed):
    edges = O.chung_lu_edges(n, e, exponent=0.8, seed=seed)
    g = pgl.Graph(edges=edges, num_nodes=n + EMPTY)
    g.tensor()
    return g


def _rand(shape, dtype, seed):
    return torch.randn(shape, device="cuda", generator=torch.Generator("cuda").manual_seed(seed)).to(dtype)


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


@pytest.fixture(scope="module")
def hub_graph(pgl):
    g = _graph(pgl, 4000, 80000, seed=11)
    fwd = g._fwd_csr()
    deg = (fwd["indptr"][1:] - fwd["indptr"][:-1]).cpu().numpy()
    assert deg.max() > 1024 and (deg == 0).sum() >= EMPTY   # hub rows and empty rows
    return g


# 1. bit-exact against the sequential oracle ------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [4, 32, 64, 96, 100, 128, 200])
def test_unscaled_bit_exact_against_oracle(pgl, hub_graph, oracle_c, dtype, D):
    import ctypes
    from pgl_b200 import ops
    fwd = hub_graph._fwd_csr()
    N = int(hub_graph.num_nodes)
    x = _rand((N, D), dtype, D)
    x32 = np.ascontiguousarray(x.float().cpu().numpy())
    indptr = fwd["indptr"].cpu().numpy()
    cols = fwd["cols"].cpu().numpy()
    short = torch.from_numpy(np.diff(indptr) <= 1024)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    for op_i, op_ in enumerate(("sum", "mean", "max", "min")):
        ref = np.empty((N, D), np.float32)
        assert oracle_c.orc_send_u_recv_csr_f32(p(x32), p(indptr), p(cols), ctypes.c_int64(N), ctypes.c_int64(D),
                                                op_i, p(ref), 4) == 0
        out = ops.aggregate_copy(x, fwd, N, op_)
        assert out.dtype == dtype
        ref_t = torch.from_numpy(ref)
        want = ref_t.to(dtype)
        got = out.cpu()
        assert torch.equal(_bits(got[short]), _bits(want[short])), (op_, D)
        assert _within_bar(got[~short], ref_t[~short], dtype), (op_, D)


# 2. bit-exact on the wide-row path against the fp32 library --------------------------------------------------------
def _packings(ops, cols, n_src):
    packs = {name: tuple(ops.pack_cols(cols, n_src, 256, budget_bytes=b))
             for name, b in (("none", 0), ("few", 8 * 256), ("mixed", 1 << 19))}
    assert not packs["none"][1] and packs["few"][1] and packs["mixed"][1]
    packs["all"] = (cols.to(torch.int32) | -(1 << 31), True)
    return packs


def _wide_row_report():
    """(mismatches against round16 of the fp32 library, case -> 16-bit output digest)."""
    import hashlib
    import pgl_b200 as pgl
    import pgl_b200.nn.functional as GF
    from pgl_b200 import ops
    bad, digests = [], {}
    for avg_deg in (5, 15):               # both ring geometries of spmm_v5
        g = _graph(pgl, 20000, 20000 * avg_deg, seed=avg_deg)
        N = int(g.num_nodes)
        fwd = g._fwd_csr()
        norm = GF.degree_norm(g).reshape(-1)
        assert fwd["slot_scale"](norm) is None and fwd["slot_scale"](norm) is not None
        packs = _packings(ops, fwd["cols"], N)
        for D in (128, 96):
            x32 = torch.randn(N, D, device="cuda", generator=torch.Generator("cuda").manual_seed(D + avg_deg))
            for case in ("sum", "mean", "gcn_gathered", "gcn_streamed"):
                for name, pk in packs.items():
                    kw = dict(max_degree=fwd["max_degree"], packed=pk)
                    if case.startswith("gcn"):
                        kw.update(scale_src=norm, scale_dst=norm)
                        if case == "gcn_streamed":
                            kw["packed"] = ops.PackedCols(pk, fwd["slot_scale"])
                    reduce_op = "mean" if case == "mean" else "sum"
                    for dtype in DTYPES:
                        x = x32.to(dtype)
                        out = ops._spmm_raw(fwd["indptr"], fwd["cols"], x, N, reduce_op, **kw)
                        ref = ops._spmm_raw(fwd["indptr"], fwd["cols"], x.float(), N, reduce_op, **kw).to(dtype)
                        key = "deg%d/D%d/%s/%s/%s" % (avg_deg, D, case, name, str(dtype))
                        if out.dtype != dtype or not torch.equal(_bits(out), _bits(ref)):
                            bad.append(key)
                        digests[key] = hashlib.sha256(_bits(out).cpu().numpy().tobytes()).hexdigest()
    return bad, digests


def _child(env):
    code = ("import sys, json; sys.path[:0] = [%r, %r]; import test_gpu_half as t; "
            "print(json.dumps(t._wide_row_report()))" % (ROOT, HERE))
    r = subprocess.run([sys.executable, "-s", "-c", code], env=dict(os.environ, **env), capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    return json.loads(r.stdout.strip().splitlines()[-1])


def _agree_across_packings(digests):
    by_case = {}
    for key, d in digests.items():
        case = key.split("/")
        by_case.setdefault("/".join(case[:3] + case[4:]), set()).add(d)
    return {k: v for k, v in by_case.items() if len(v) != 1}


def test_wide_rows_bit_identical_to_rounded_fp32():
    """Every packing, both geometries, both norms: round16(fp32) bit for bit, and every packing agrees."""
    bad, mine = _wide_row_report()
    assert bad == []
    assert _agree_across_packings(mine) == {}


def test_wide_rows_bit_identical_with_short_tasks():
    """64-slot tasks cut hub rows into fp32 partials that the 16-bit fix-up kernel adds and rounds once."""
    bad, short = _child({"PGLB_STREAM_TASK": "64"})
    assert bad == [] and _agree_across_packings(short) == {}


# 3. the bar for scaled calls on the node-parallel kernel and cut hub rows -------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [4, 32, 100, 200])
def test_scaled_generic_within_bar(pgl, hub_graph, dtype, D):
    import pgl_b200.nn.functional as GF
    from pgl_b200 import ops
    fwd = hub_graph._fwd_csr()
    N = int(hub_graph.num_nodes)
    norm = GF.degree_norm(hub_graph).reshape(-1)
    x = _rand((N, D), dtype, 3 * D)
    a = sp.csr_matrix((np.ones(int(fwd["cols"].shape[0])), fwd["cols"].cpu().numpy(), fwd["indptr"].cpu().numpy()),
                      shape=(N, N))
    s = norm.double().cpu().numpy()[:, None]
    ref = (a @ (x.double().cpu().numpy() * s)) * s
    for scale in (norm, norm.to(dtype)):    # a 16-bit norm is widened to fp32 first
        out = ops.aggregate_copy(x, fwd, N, "sum", scale_src=scale, scale_dst=scale)
        assert out.dtype == dtype
        s16 = scale.double().cpu().numpy()[:, None]
        want = ref if scale.dtype == torch.float32 else (a @ (x.double().cpu().numpy() * s16)) * s16
        assert _within_bar(out, want, dtype)


# 4. autograd --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_gradients_within_bar(pgl, dtype):
    from pgl_b200.nn.conv import _propagate
    import pgl_b200.nn.functional as GF
    g = _graph(pgl, 3000, 30000, seed=4)
    N = int(g.num_nodes)
    norm = GF.degree_norm(g).reshape(-1, 1)
    for D in (32, 128):
        x0 = _rand((N, D), dtype, D)
        up = _rand((N, D), dtype, D + 1)
        fns = {op_: (lambda x, op_=op_: g.send_recv(x, op_)) for op_ in ("sum", "mean", "max", "min")}
        fns["gcn"] = lambda x: _propagate(g, x, norm)
        for name, fn in fns.items():
            x = x0.clone().requires_grad_()
            out = fn(x)
            assert out.dtype == dtype
            out.backward(up)
            x32 = x0.float().requires_grad_()
            fn(x32).backward(up.float())
            assert x.grad.dtype == dtype
            assert _within_bar(x.grad, x32.grad, dtype), (name, D)


# 5. layers ----------------------------------------------------------------------------------------------------------
def _layers(pgl):
    nn = pgl.nn
    return {
        "gcn": lambda: nn.GCNConv(128, 96),
        "sage_sum": lambda: nn.GraphSageConv(96, 64, "sum"),
        "sage_mean": lambda: nn.GraphSageConv(96, 64, "mean"),
        "sage_max": lambda: nn.GraphSageConv(96, 64, "max"),
        "gat": lambda: nn.GATConv(96, 32, feat_drop=0.0, attn_drop=0.0, num_heads=4),
        "appnp": lambda: nn.APPNP(alpha=0.2, k_hop=4),
    }


def _normwise(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("name", ["gcn", "sage_sum", "sage_mean", "sage_max", "gat", "appnp"])
def test_layers_bf16(pgl, monkeypatch, name):
    from pgl_b200 import ops
    calls = []
    real = ops.lib.pglb_spmm_csr_x16

    def spy(*a):
        calls.append(a[10])
        return real(*a)

    monkeypatch.setattr(ops.lib, "pglb_spmm_csr_x16", spy)
    g = _graph(pgl, 3000, 30000, seed=8)
    N = int(g.num_nodes)
    din = 128 if name == "gcn" else 96
    torch.manual_seed(0)
    ref_layer = _layers(pgl)[name]().cuda()
    x = torch.randn(N, din, device="cuda")
    x32 = x.clone().requires_grad_()
    ref = ref_layer(g, x32)
    ref.backward(torch.ones_like(ref))
    # autocast: fp32 parameters, 16-bit activations where torch makes them
    layer = _layers(pgl)[name]().cuda()
    layer.load_state_dict(ref_layer.state_dict())
    xa = x.clone().requires_grad_()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out = layer(g, xa)
    out.float().backward(torch.ones_like(out, dtype=torch.float32))
    assert _normwise(out, ref) <= 3e-2 and _normwise(xa.grad, x32.grad) <= 3e-2
    # the whole module in bf16
    layer16 = _layers(pgl)[name]().cuda()
    layer16.load_state_dict(ref_layer.state_dict())
    layer16 = layer16.to(torch.bfloat16)
    x16 = x.to(torch.bfloat16).requires_grad_()
    out16 = layer16(g, x16)
    assert out16.dtype == torch.bfloat16
    out16.backward(torch.ones_like(out16))
    assert x16.grad.dtype == torch.bfloat16
    assert _normwise(out16, ref) <= 3e-2 and _normwise(x16.grad, x32.grad) <= 3e-2
    if name in ("gcn", "appnp", "sage_sum", "sage_mean", "sage_max"):
        assert ops._lib.DTYPE_BF16 in calls   # the aggregation ran on the native 16-bit entry


# 6. training --------------------------------------------------------------------------------------------------------
def test_cora_training_under_bf16_autocast(pgl):
    from test_gpu_cora import GCN
    cora = O.load_cora(os.path.join(HERE, "golden", "cora.npz"))
    n = cora["num_nodes"]
    g = pgl.Graph(edges=cora["edges"], num_nodes=n)
    g.tensor()
    x = torch.from_numpy(cora["x"]).cuda()
    y = torch.from_numpy(cora["y"]).cuda()
    idx = {k: torch.from_numpy(cora[k + "_index"]).cuda() for k in ("train", "val", "test")}
    torch.manual_seed(0)
    model = GCN(pgl, 1433, cora["num_classes"]).cuda()
    optim = torch.optim.Adam(model.parameters(), lr=0.01, weight_decay=5e-4)
    loss_fn = torch.nn.CrossEntropyLoss()
    best_val, test_at_best = -1.0, 0.0
    for epoch in range(200):
        model.train()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            pred = model(g, x)
            loss = loss_fn(pred[idx["train"]].float(), y[idx["train"]])
        optim.zero_grad()
        loss.backward()
        optim.step()
        model.eval()
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            pred = model(g, x).argmax(1)
            val = float((pred[idx["val"]] == y[idx["val"]]).float().mean())
            test = float((pred[idx["test"]] == y[idx["test"]]).float().mean())
        if val > best_val:
            best_val, test_at_best = val, test
    assert 0.77 <= test_at_best <= 0.85, (best_val, test_at_best)


# 7. ops without 16-bit kernels: widened to fp32, rounded back ---------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_widen_through_ops(pgl, dtype):
    import pgl_b200.nn.functional as GF
    g = _graph(pgl, 2000, 16000, seed=9)
    N, E = int(g.num_nodes), int(g.num_edges)
    x = _rand((N, 64), dtype, 1)
    y = _rand((N, 64), dtype, 2)
    w = _rand((E, 1), dtype, 3)
    logits = _rand((E, 4), dtype, 4)
    seg = torch.sort(g.edges[:, 1])[0]     # sorted segment ids, with gaps

    def udf_send(src, dst, edge):
        return {"m": src["h"] * 2.0}

    cases = {
        "send_ue_recv": lambda a, b, c, l: g.send_ue_recv(a, c, "mul", "sum"),
        "send_uv": lambda a, b, c, l: g.send_uv(a, b, "add"),
        "edge_softmax": lambda a, b, c, l: GF.edge_softmax(g, l),
        "segment_softmax": lambda a, b, c, l: pgl.math.segment_softmax(l, seg),
        "udf": lambda a, b, c, l: g.recv(lambda m: m.reduce_sum(m["m"]),
                                         g.send(udf_send, src_feat={"h": a})),
    }
    for name, fn in cases.items():
        out = fn(x, y, w, logits)
        ref = fn(x.float(), y.float(), w.float(), logits.float())
        assert out.dtype == dtype, name
        assert _within_bar(out, ref, dtype), name
    # bf16 with fp32 promotes to fp32; float64 follows the float64 rule
    assert g.send_uv(x, y.float(), "add").dtype == torch.float32
    assert g.send_ue_recv(x, w.float(), "mul", "sum").dtype == torch.float32
    assert g.send_uv(x, y.double(), "add").dtype == torch.float64


@pytest.mark.parametrize("dtype", DTYPES)
def test_segment_gradients_within_bar(pgl, dtype):
    """segment_* (identity slots), the fused-gather segment reduce and the UDF send -> recv reduce: the 16-bit
    gradient is formed in fp32 and rounded once, so it meets the bar against the fp32 backward on widened inputs."""
    from pgl_b200 import ops
    g = _graph(pgl, 2000, 40000, seed=12)
    N, E = int(g.num_nodes), int(g.num_edges)
    ids = torch.sort(g.edges[:, 1])[0]                  # sorted segment ids with gaps; hub segments > 1024 slots
    fwd = g._fwd_csr()
    assert int(fwd["max_degree"]) > 1024
    data0 = _rand((E, 32), dtype, 5)
    x0 = _rand((N, 32), dtype, 6)

    def udf(red):
        return lambda x: g.recv(lambda m: getattr(m, red)(m["m"]), g.send(lambda s, d, e: {"m": s["h"]}, src_feat={"h": x}))

    cases = {"segment_" + op_: (data0, lambda d, op_=op_: getattr(pgl.math, "segment_" + op_)(d, ids))
             for op_ in ("sum", "mean", "max", "min")}
    for op_ in ("sum", "mean"):
        cases["gather_" + op_] = (x0, lambda x, op_=op_: ops.segment_reduce(
            x, None, op_, indptr=fwd["indptr"], cols=fwd["cols"], max_degree=fwd["max_degree"]))
        cases["udf_" + op_] = (x0, udf("reduce_" + op_))
    for name, (inp, fn) in cases.items():
        x = inp.clone().requires_grad_()
        out = fn(x)
        assert out.dtype == dtype, name
        up = _rand(tuple(out.shape), dtype, 7)
        out.backward(up)
        x32 = inp.float().requires_grad_()
        fn(x32).backward(up.float())
        assert x.grad.dtype == dtype, name
        assert _within_bar(x.grad, x32.grad, dtype), name


@pytest.mark.parametrize("dtype", DTYPES)
def test_segment_mean_gradient_of_a_long_segment(pgl, dtype):
    """A segment longer than float16's largest finite value (65504): the count stays exact in fp32, so the mean's
    gradient is g / count, not 0."""
    L = 70000
    ids = torch.cat([torch.zeros(L, dtype=torch.int64), torch.ones(3, dtype=torch.int64)]).cuda()
    x = _rand((L + 3, 4), dtype, 8).requires_grad_()
    out = pgl.math.segment_mean(x, ids)
    up = torch.ones_like(out)
    out.backward(up)
    want = torch.cat([torch.full((L, 4), 1.0 / L), torch.full((3, 4), 1.0 / 3)]).cuda()
    assert x.grad.dtype == dtype and _within_bar(x.grad, want, dtype)
    assert float(x.grad[:L].float().min()) > 0


def test_fp32_route_widens_16bit_norms(pgl):
    """fp32 features with a 16-bit norm: the norm is widened to fp32 before the fp32 entry reads it."""
    from pgl_b200 import ops
    import pgl_b200.nn.functional as GF
    g = _graph(pgl, 2000, 16000, seed=13)
    N = int(g.num_nodes)
    fwd = g._fwd_csr()
    norm = GF.degree_norm(g).reshape(-1).to(torch.bfloat16)
    x = _rand((N, 32), torch.float32, 9)
    out = ops.aggregate_copy(x, fwd, N, "sum", scale_src=norm, scale_dst=norm)
    want = ops.aggregate_copy(x, fwd, N, "sum", scale_src=norm.float(), scale_dst=norm.float())
    assert out.dtype == torch.float32 and torch.equal(out, want)
