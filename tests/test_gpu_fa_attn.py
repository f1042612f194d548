"""FAConv's fused self-gated aggregation (pglb_fa_attn_*, pglb_fa_bwd_edge_*, ops.fa_attention, FAConv).

Contract: for dst row d and the in-edges e = (u -> d) of d, t_e = tanh(g_src[u] + g_dst[d]),
w_e = keep_e s ((t_e norm[u]) norm[d]), out[d] = sum_e w_e f[u] (rows without in-edges: 0).  Without dropout
keep_e s = 1; with dropout keep_e is bit 0 of GAT's 4-head keep word of the edge's dst-CSR slot and s = 1 / (1 - p).
The references are torch restatements of that contract: float64 for the float32 kernels, the float32 kernels on widened
inputs for the 16-bit ones (bit for bit), plain torch fp32 with the library's mask for dropout."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

from oracle import oracle as O
from test_gpu_exact_routes import _kernels_of

pytestmark = pytest.mark.gpu
DIMS = [4, 8, 16, 24, 64, 100, 128]
DIMS16 = [8, 16, 24, 64, 128]
DTYPES = (torch.bfloat16, torch.float16)
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
EMPTY = 64   # trailing nodes without an edge: empty rows
SEED = (0x5EED0123456789AB, 4 * 1000)
GRAD_TOL = 2e-4   # float32 gradients against float64 autograd, relative to the largest |grad|
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
FA_FWD = re.compile(r"spmm_gat5_kernel<[^>]*, (true|false), 4>")


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


@pytest.fixture(scope="module")
def graph(pgl):
    """Rows cut across tasks (in-degree > 2048: the fix-up path), one-edge rows, empty rows, multi-edges, self-loops,
    and edge ids that differ from the dst-CSR slots."""
    n = 3000
    edges = O.chung_lu_edges(n, 80000, exponent=0.9, seed=401)
    g = pgl.Graph(edges=edges, num_nodes=n + EMPTY)
    g.tensor()
    deg = np.bincount(edges[:, 1], minlength=n + EMPTY)
    assert deg.max() > 2048 and (deg == 0).sum() >= EMPTY and (deg == 1).sum() > 0
    assert (edges[:, 0] == edges[:, 1]).any() and len(np.unique(edges, axis=0)) < len(edges)
    eid = g._fwd_csr()["eid"]
    assert not torch.equal(eid, torch.arange(len(edges), device=eid.device))
    return g, edges


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _rand(shape, seed, dtype=torch.float32, scale=1.0):
    g = torch.Generator("cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


def _gates(N, seed, dtype=torch.float32):
    """g_src, g_dst [N, 1]: most |g_src + g_dst| between 0 and ~12 (tanh saturates), every fifth node near 0."""
    gs, gd = _rand((N, 1), seed, scale=3.0), _rand((N, 1), seed + 1, scale=3.0)
    gs[::5] *= 1e-3
    gd[::5] *= 1e-3
    return gs.to(dtype), gd.to(dtype)


def _inputs(g, D, seed, dtype=torch.float32):
    N = g.num_nodes
    f = _rand((N, D), seed, dtype)
    gs, gd = _gates(N, seed + 1, dtype)
    from pgl_b200.nn import functional as GF
    return f, gs, gd, GF.degree_norm(g)


def rel_err(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-12))


def restate(f, gs, gd, nm, src, dst, mask=None, s=1.0):
    """The contract in torch, differentiable, in f's dtype."""
    t = torch.tanh(gs.reshape(-1)[src] + gd.reshape(-1)[dst])
    w = (t * nm.reshape(-1)[src].to(t.dtype)) * nm.reshape(-1)[dst].to(t.dtype)
    if mask is not None:
        w = w * mask * torch.tensor(s, dtype=w.dtype, device=w.device)
    return torch.zeros_like(f).index_add(0, dst, f[src] * w.unsqueeze(-1))


def edge_mask(csr, p, seed=SEED):
    """[E] float32 keep mask in edge order: bit 0 of the 4-head keep word of each dst-CSR slot."""
    from pgl_b200 import _lib
    E = int(csr["cols"].shape[0])
    w = np.zeros(E, np.uint32)
    _lib.check(_lib.lib.pglb_attn_dropout_keep_host(seed[0], seed[1], p, 0, E, 4, w.ctypes.data_as(ctypes.c_void_p)))
    m = np.empty(E, np.float32)
    m[csr["eid"].cpu().numpy()] = (w & 1).astype(np.float32)
    return torch.from_numpy(m).cuda()


def _s32(p):
    return float(np.float32(1.0 / (1.0 - float(np.float32(p)))))


def fwd_raw(pgl, csr, f, gs, gd, nm, drop=None):
    ops = pgl.ops
    return ops._fa_fwd_raw(csr, f, ops._fa_records(gs.reshape(-1), nm.reshape(-1), gd.reshape(-1)), drop)


def bwd_raw(pgl, csr, f, gs, gd, nm, go, drop=None):
    """The edge backward entry of f's dtype: (beta_e, dz_e)."""
    ops = pgl.ops
    rec = ops._fa_records(gs.reshape(-1), nm.reshape(-1), gd.reshape(-1))
    E, D = int(csr["cols"].shape[0]), int(f.shape[1])
    beta = torch.empty(E, device="cuda")
    dz = torch.empty(E, device="cuda")
    dt = () if f.dtype == torch.float32 else (ops._DTYPE16[f.dtype],)
    name = "pglb_fa_bwd_edge_%s%s" % ("drop_" if drop else "", "x16" if dt else "f32")
    ops.check(getattr(ops.lib, name)(
        ops._ptr(csr["rows"]), ops._ptr(csr["cols"]), ops._ptr(csr["eid"]), ops._ptr(f), f.stride(0), ops._ptr(rec),
        ops._ptr(go), go.stride(0), E, D, *dt, *(drop or ()), ops._ptr(beta), ops._ptr(dz), ops._stream()))
    return beta, dz


def _ends(edges):
    return torch.from_numpy(edges[:, 0]).cuda(), torch.from_numpy(edges[:, 1]).cuda()


@pytest.mark.parametrize("D", DIMS)
def test_forward_against_float64(pgl, graph, D):
    g, edges = graph
    src, dst = _ends(edges)
    f, gs, gd, nm = _inputs(g, D, 10 + D)
    assert float((gs[src] + gd[dst]).abs().max()) > 9.0 and float((gs[src] + gd[dst]).abs().min()) < 1e-2
    out = fwd_raw(pgl, g._fwd_csr(), f, gs, gd, nm)
    again = fwd_raw(pgl, g._fwd_csr(), f, gs, gd, nm)
    assert torch.equal(_bits(out), _bits(again))
    want = restate(f.double(), gs.double(), gd.double(), nm.double(), src, dst)
    assert (out[-EMPTY:] == 0).all()
    assert float((out.double() - want).abs().max()) <= 1e-4 * float(want.abs().max())
    # the public call without autograd: the same entry, the same bits
    inf = pgl.ops.fa_attention(g._fwd_csr(), g._bwd_csr, f, gs, gd, nm)
    assert inf.dtype == torch.float32 and torch.equal(_bits(inf), _bits(out))


def _grad_check(pgl, g, edges, f, gs, gd, nm):
    src, dst = _ends(edges)
    f, gs, gd = (t.clone().requires_grad_() for t in (f, gs, gd))
    go = _rand(f.shape, 5)
    out = pgl.ops.fa_attention(g._fwd_csr(), g._bwd_csr, f, gs, gd, nm)
    got = torch.autograd.grad(out, (f, gs, gd), go)
    ins = [t.detach().double().requires_grad_() for t in (f, gs, gd)]
    want = torch.autograd.grad(restate(*ins, nm.double(), src, dst), ins, go.double())
    for name, x, y in zip(("f", "g_src", "g_dst"), got, want):
        assert x.dtype == torch.float32 and x.shape == y.shape and rel_err(x, y) <= GRAD_TOL, (name, rel_err(x, y))
    return got


@pytest.mark.parametrize("D", DIMS)
def test_gradients_against_float64_autograd(pgl, graph, D):
    g, edges = graph
    f, gs, gd, nm = _inputs(g, D, 20 + D)
    got = _grad_check(pgl, g, edges, f, gs, gd, nm)
    again = _grad_check(pgl, g, edges, f, gs, gd, nm)   # no floating-point atomics: identical bits
    for x, y in zip(got, again):
        assert torch.equal(_bits(x), _bits(y))
    # [N] gates give [N] gradients
    g1 = _grad_check(pgl, g, edges, f, gs.reshape(-1), gd.reshape(-1), nm.reshape(-1))
    assert g1[1].shape == (g.num_nodes,) and torch.equal(_bits(g1[1]), _bits(got[1].reshape(-1)))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", DIMS16)
def test_x16_bit_exact_against_fp32_kernel(pgl, graph, dtype, D):
    g, _ = graph
    fwd = g._fwd_csr()
    f, gs, gd, nm = _inputs(g, D, 30 + D, dtype)
    for drop in (None, (0.4,) + SEED):
        out16 = fwd_raw(pgl, fwd, f, gs, gd, nm, drop)
        out32 = fwd_raw(pgl, fwd, f.float(), gs, gd, nm, drop)
        assert out16.dtype == dtype and torch.equal(_bits(out16), _bits(out32.to(dtype)))
        go = _rand(f.shape, 7, dtype)
        r16 = bwd_raw(pgl, fwd, f, gs, gd, nm, go, drop)
        r32 = bwd_raw(pgl, fwd, f.float(), gs, gd, nm, go.float(), drop)
        for x, y in zip(r16, r32):
            assert torch.equal(_bits(x), _bits(y))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("D", [8, 24, 128])
def test_x16_gradients_against_fp32_autograd(pgl, graph, dtype, D):
    """16-bit gradients are fp32 sums rounded once to the input's dtype: within 2 u of the largest |grad| of fp32 torch
    autograd on the widened inputs."""
    g, edges = graph
    src, dst = _ends(edges)
    f, gs, gd, nm = _inputs(g, D, 40 + D, dtype)
    f, gs, gd = (t.requires_grad_() for t in (f, gs, gd))
    go = _rand(f.shape, 9, dtype)
    out = pgl.ops.fa_attention(g._fwd_csr(), g._bwd_csr, f, gs, gd, nm)
    assert out.dtype == dtype
    got = torch.autograd.grad(out, (f, gs, gd), go)
    ins = [t.detach().float().requires_grad_() for t in (f, gs, gd)]
    want = torch.autograd.grad(restate(*ins, nm, src, dst), ins, go.float())
    for name, x, y in zip(("f", "g_src", "g_dst"), got, want):
        assert x.dtype == dtype and rel_err(x, y) <= 2 * U[dtype], (name, rel_err(x, y))


@pytest.mark.parametrize("D", [8, 24, 64])
def test_dropout(pgl, graph, D):
    g, edges = graph
    fwd = g._fwd_csr()
    src, dst = _ends(edges)
    p = 0.6
    drop = (p,) + SEED
    mask, s = edge_mask(fwd, p), _s32(p)
    assert 0.3 < float(mask.mean()) < 0.5
    f, gs, gd, nm = _inputs(g, D, 50 + D)
    out = fwd_raw(pgl, fwd, f, gs, gd, nm, drop)
    assert torch.equal(_bits(out), _bits(fwd_raw(pgl, fwd, f, gs, gd, nm, drop)))   # same (seed, offset), same bits
    other = fwd_raw(pgl, fwd, f, gs, gd, nm, (p, SEED[0], SEED[1] + 4))
    assert not torch.equal(other, out)
    out0 = fwd_raw(pgl, fwd, f, gs, gd, nm)
    tiny = fwd_raw(pgl, fwd, f, gs, gd, nm, (1e-12,) + SEED)   # p = 1e-12 keeps every slot with s = 1
    assert torch.equal(_bits(tiny), _bits(out0))
    assert rel_err(out, restate(f, gs, gd, nm, src, dst, mask, s)) <= 1e-4
    # the backward recomputes the same mask from (seed, offset): gradients against torch fp32 with that mask
    ins = [t.clone().requires_grad_() for t in (f, gs, gd)]
    go = _rand(f.shape, 13)
    o = pgl.ops.fa_attention(fwd, g._bwd_csr, *ins, nm, attn_drop=p, seed=SEED)
    assert torch.equal(_bits(o.detach()), _bits(out))
    got = torch.autograd.grad(o, ins, go)
    ref = [t.clone().requires_grad_() for t in (f, gs, gd)]
    want = torch.autograd.grad(restate(*ref, nm, src, dst, mask, s), ref, go)
    for name, x, y in zip(("f", "g_src", "g_dst"), got, want):
        assert rel_err(x, y) <= GRAD_TOL, (name, rel_err(x, y))
    b_tiny = bwd_raw(pgl, fwd, f, gs, gd, nm, go, (1e-12,) + SEED)
    b0 = bwd_raw(pgl, fwd, f, gs, gd, nm, go)
    for x, y in zip(b_tiny, b0):
        assert torch.equal(_bits(x), _bits(y))


def test_layer_dropout_replays_under_manual_seed(pgl, graph):
    g, _ = graph
    conv = pgl.nn.FAConv(24, drop=0.5).cuda().train()
    x = _rand((g.num_nodes, 24), 55)
    calls = []
    real = pgl.ops.fa_attention

    def counted(*a, **kw):
        r = real(*a, **kw)
        calls.append(r is not None)
        return r
    pgl.ops.fa_attention = counted
    try:
        torch.manual_seed(5)
        a = conv(g, x)
        b = conv(g, x)
        torch.manual_seed(5)
        c = conv(g, x)
    finally:
        pgl.ops.fa_attention = real
    assert calls == [True] * 3
    assert torch.equal(_bits(a), _bits(c)) and not torch.equal(a, b)


def test_calls_outside_the_kernels_return_none(pgl, graph):
    g, _ = graph
    N = g.num_nodes
    fwd, bwd = g._fwd_csr(), g._bwd_csr
    fa = pgl.ops.fa_attention
    f, gs, gd, nm = _inputs(g, 24, 61)
    assert fa(fwd, bwd, f, gs, gd, nm) is not None
    assert fa(fwd, bwd, f.double(), gs, gd, nm) is None                          # float64 anywhere
    assert fa(fwd, bwd, f, gs.double(), gd, nm) is None and fa(fwd, bwd, f, gs, gd, nm.double()) is None
    assert fa(fwd, bwd, f.bfloat16(), gs, gd, nm) is None                         # dtype mix: the result would be fp32
    assert fa(fwd, bwd, f.bfloat16(), gs.half(), gd.half(), nm) is None
    assert fa(fwd, bwd, f.bfloat16(), gs.bfloat16(), gd.bfloat16(), nm, out_dtype=torch.float32) is None
    assert fa(fwd, bwd, _rand((N, 132), 62), gs, gd, nm) is None                  # D > 128
    assert fa(fwd, bwd, _rand((N, 130), 62), gs, gd, nm) is None
    assert fa(fwd, bwd, _rand((N, 6), 63), gs, gd, nm) is None                    # 24-byte rows
    assert fa(fwd, bwd, _rand((N, 12), 64, torch.bfloat16), gs.bfloat16(), gd.bfloat16(), nm) is None
    assert fa(fwd, bwd, f, gs, gd, nm.clone().requires_grad_()) is None           # norm is a constant
    assert fa(fwd, bwd, f[:-1], gs[:-1], gd[:-1], nm[:-1]) is None               # n_dst != N
    assert fa(dict(fwd, cols=fwd["cols"][:0]), bwd, f, gs, gd, nm) is None       # no edges
    assert fa(fwd, bwd, f, gs, gd, nm, attn_drop=1.0) is None and fa(fwd, bwd, f, gs, gd, nm, attn_drop=1.5) is None
    buf = torch.empty(N * 24 + 1, device="cuda")
    mis = buf[1:].view(N, 24)
    mis.copy_(f)
    assert fa(fwd, bwd, mis, gs, gd, nm) is None                                  # f not 16-byte aligned
    assert fa({k_: v_ for k_, v_ in fwd.items() if k_ != "rows"}, bwd, f, gs, gd, nm) is None
    graph_ = torch.cuda.CUDAGraph()
    res = []
    with torch.cuda.graph(graph_):
        res.append(fa(fwd, bwd, f, gs, gd, nm, attn_drop=0.5))                    # dropout during capture
    assert res == [None]


def _op_by_op(conv, g, x):
    """FAConv.forward through the op-by-op route (send_uv(add), tanh, send_uv(norm, norm, mul), dropout,
    send_ue_recv)."""
    from pgl_b200.nn import functional as GF
    norm = GF.degree_norm(g)
    d = conv.hidden_size
    g_src = x @ conv.gate.weight[:d]
    g_dst = x @ conv.gate.weight[d:] + conv.gate.bias
    h = torch.tanh(g.send_uv(g_src, g_dst, "add"))
    alpha = conv.dropout(h * g.send_uv(norm, norm, "mul"))
    return g.send_ue_recv(x, alpha, "mul", "sum")


@pytest.mark.parametrize("mode", ["eval", "train"])
def test_layer_matches_op_by_op_with_fewer_launches(pgl, graph, mode):
    g, _ = graph
    N, D = g.num_nodes, 24
    torch.manual_seed(3)
    conv = pgl.nn.FAConv(D, drop=0.0).cuda()
    conv.train(mode == "train")
    x = _rand((N, D), 71).requires_grad_()
    go = _rand((N, D), 72)
    params = [x] + list(conv.parameters())
    conv(g, x).square().sum().backward()          # warm: CSRs, norms and workspaces outside the profiled calls
    fused_names, fused = _kernels_of(lambda: torch.autograd.grad(conv(g, x), params, go))
    opby_names, _ = _kernels_of(lambda: torch.autograd.grad(_op_by_op(conv, g, x), params, go))
    if not opby_names:
        pytest.skip("torch.profiler records no CUDA kernels here")
    assert any(FA_FWD.search(n) for n in fused_names), fused_names
    assert any("fa_bwd_edge_kernel" in n for n in fused_names), fused_names
    assert not any(FA_FWD.search(n) or "fa_bwd_edge_kernel" in n for n in opby_names)
    assert len(fused_names) < len(opby_names), (len(fused_names), len(opby_names))
    out = conv(g, x)
    got = torch.autograd.grad(out, params, go)
    ref = _op_by_op(conv, g, x)
    want = torch.autograd.grad(ref, params, go)
    assert out.dtype == ref.dtype and rel_err(out, ref) <= 1e-4
    for name, a, b in zip(["x"] + [n for n, _ in conv.named_parameters()], got, want):
        assert a.dtype == b.dtype and a.shape == b.shape and rel_err(a, b) <= 1e-4, (name, rel_err(a, b))
    with torch.no_grad():   # inference reaches the forward entry without autograd
        assert rel_err(conv(g, x), ref) <= 1e-4


def test_layer_16bit_keeps_the_op_by_op_dtypes(pgl, graph):
    """A bfloat16 layer: the op-by-op route returns float32 (the norms are float32); the fused route aggregates on the
    16-bit kernel and returns the same dtype, with gradients in each input's dtype."""
    g, _ = graph
    N, D = g.num_nodes, 16
    torch.manual_seed(4)
    conv = pgl.nn.FAConv(D, drop=0.0).cuda().to(torch.bfloat16)
    x = _rand((N, D), 73, torch.bfloat16).requires_grad_()
    params = [x] + list(conv.parameters())
    names, _ = _kernels_of(lambda: conv(g, x))
    out = conv(g, x)
    ref = _op_by_op(conv, g, x)
    assert out.dtype == ref.dtype == torch.float32 and rel_err(out, ref) <= 4 * U[torch.bfloat16]
    got = torch.autograd.grad(out.sum(), params)
    want = torch.autograd.grad(ref.sum(), params)
    for a, b in zip(got, want):
        assert a.dtype == b.dtype and rel_err(a, b) <= 0.05
    assert any(FA_FWD.search(n) for n in names) or not names, names


@pytest.mark.parametrize("D,dtype", [(130, torch.float32), (24, torch.float64)])
def test_declined_layer_keeps_the_op_by_op_output(pgl, graph, D, dtype):
    g, _ = graph
    torch.manual_seed(6)
    conv = pgl.nn.FAConv(D, drop=0.0).cuda().to(dtype).eval()
    x = _rand((g.num_nodes, D), 74).to(dtype)
    with torch.no_grad():
        assert torch.equal(conv(g, x), _op_by_op(conv, g, x))


def test_layer_memory_has_no_edge_tensor(pgl):
    """One [E] float32 tensor is 8 MB here: a forward under autograd allocates less than that (autograd keeps only
    N-sized tensors), and the forward + backward peak is below the op-by-op route's."""
    n, e, D = 20000, 2_000_000, 16
    edges = O.chung_lu_edges(n, e, exponent=0.8, seed=81)
    g = pgl.Graph(edges=edges, num_nodes=n)
    g.tensor()
    conv = pgl.nn.FAConv(D, drop=0.0).cuda()
    x = _rand((n, D), 82).requires_grad_()
    conv(g, x).sum().backward()                   # warm: CSRs, norms, workspaces
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    out = conv(g, x)
    grown = torch.cuda.memory_allocated() - base
    del out
    assert grown < e * 4, (grown, e * 4)

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        b = torch.cuda.memory_allocated()
        fn(g, x).square().sum().backward()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - b

    fused = peak(conv)
    opby = peak(lambda gg, xx: _op_by_op(conv, gg, xx))
    assert fused < opby, (fused, opby)


class _FAGCN(torch.nn.Module):
    """The reference's examples/fagcn model: dropout, Linear + relu, dropout, num_layer FAConv layers each followed by
    eps * h0 + h, Linear."""

    def __init__(self, pgl, input_size, hidden_size, output_size, drop=0.6, eps=0.2, num_layer=5):
        super().__init__()
        self.dropout = torch.nn.Dropout(p=drop)
        self.eps = eps
        self.gnn_layer = torch.nn.ModuleList([pgl.nn.FAConv(hidden_size, drop) for _ in range(num_layer)])
        self.t1 = torch.nn.Linear(input_size, hidden_size)
        self.t2 = torch.nn.Linear(hidden_size, output_size)

    def forward(self, graph, feature):
        feature = self.dropout(torch.relu(self.t1(self.dropout(feature))))
        h0 = feature
        for layer in self.gnn_layer:
            feature = self.eps * h0 + layer(graph, feature)
        return self.t2(feature)


def _train_fagcn(pgl, g, x, y, idx, classes, seed, epochs=200):
    """Test accuracy at the epoch of the lowest validation loss (the reference script's rule)."""
    torch.manual_seed(seed)
    model = _FAGCN(pgl, x.shape[1], 16, classes).cuda()
    optim = torch.optim.Adam(model.parameters(), lr=0.005, weight_decay=5e-4)
    loss_fn = torch.nn.CrossEntropyLoss()
    best_loss, test_at_best = float("inf"), 0.0
    for _ in range(epochs):
        model.train()
        loss = loss_fn(model(g, x)[idx["train"]], y[idx["train"]])
        optim.zero_grad()
        loss.backward()
        optim.step()
        model.eval()
        with torch.no_grad():
            logits = model(g, x)
        val_loss = float(loss_fn(logits[idx["val"]], y[idx["val"]]))
        if val_loss < best_loss:
            pred = logits.argmax(1)
            best_loss, test_at_best = val_loss, float((pred[idx["test"]] == y[idx["test"]]).float().mean())
    return test_at_best


def test_fagcn_trains_on_cora(pgl):
    """The reference's FAGCN (hidden 16, 5 layers, drop 0.6, eps 0.2, Adam 0.005, weight decay 5e-4, 200 epochs) on
    Cora, trained on both routes from the same seeds (the dropout masks differ: nn.Dropout against the kernels'
    stream).  The mean over three seeds of the test accuracy at the lowest validation loss must agree within 0.02 and
    clear a floor below both measured values (0.644 fused and 0.661 op by op on an H100; the example's README reports
    about 0.85 after 2000 epochs)."""
    c = O.load_cora(os.path.join(GOLDEN, "cora.npz"))
    g = pgl.Graph(edges=c["edges"], num_nodes=c["num_nodes"])
    g.tensor()
    x = torch.from_numpy(c["x"]).cuda()
    y = torch.from_numpy(c["y"]).cuda()
    idx = {k: torch.from_numpy(c[k + "_index"]).cuda() for k in ("train", "val", "test")}
    seeds = (0, 1, 2)
    calls = []
    real = pgl.ops.fa_attention

    def counted(*a, **kw):
        r = real(*a, **kw)
        calls.append(r is not None)
        return r
    pgl.ops.fa_attention = counted
    try:
        fused = float(np.mean([_train_fagcn(pgl, g, x, y, idx, c["num_classes"], s) for s in seeds]))
        assert calls and all(calls)
        pgl.ops.fa_attention = lambda *a, **kw: None
        opby = float(np.mean([_train_fagcn(pgl, g, x, y, idx, c["num_classes"], s) for s in seeds]))
    finally:
        pgl.ops.fa_attention = real
    print("fagcn cora: test accuracy at the lowest validation loss, fused %.4f, op by op %.4f" % (fused, opby))
    assert abs(fused - opby) <= 0.02, (fused, opby)
    assert min(fused, opby) >= 0.60, (fused, opby)
