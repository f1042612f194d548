"""TransformerConv's fused dot-product attention (pglb_dot_attn_*, ops.dot_attention).

Contract: for dst row d, head h and the in-edges j of d, s_j = <q[d,h,:], k[src_j,h,:]> (q already scaled),
lse = log sum_j exp(s_j), out[d,h,:] = sum_j exp(s_j - lse) v[src_j,h,:] (rows without in-edges: 0).  With dropout
(keep bits m of the GAT stream, keyed by dst-CSR slot and head; s = 1 / (1 - p)) out = sum_j s m_j a_j v_j and lse is
the value without dropout.  The references are torch restatements of that contract: float64 for the float32 kernels,
the float32 kernel on widened inputs for the 16-bit ones (bit for bit), plain torch fp32 with the library's mask for
dropout."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
LAYOUTS = [(8, 16), (4, 32), (2, 64), (8, 8), (16, 4), (32, 4), (1, 4)]
DTYPES = (torch.bfloat16, torch.float16)
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
EMPTY = 64   # trailing nodes without an edge: empty rows
SEED = (0x5EED0123456789AB, 4 * 1000)
GRAD_TOL = 2e-4   # float32 gradients against float64 autograd, relative to the largest |grad|
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


@pytest.fixture(scope="module")
def graph(pgl):
    """Rows cut across tasks (in-degree > 2048: the fix-up path), one-edge rows, empty rows, multi-edges and
    self-loops."""
    n = 3000
    edges = O.chung_lu_edges(n, 80000, exponent=0.9, seed=301)
    g = pgl.Graph(edges=edges, num_nodes=n + EMPTY)
    g.tensor()
    deg = np.bincount(edges[:, 1], minlength=n + EMPTY)
    assert deg.max() > 2048 and (deg == 0).sum() >= EMPTY and (deg == 1).sum() > 0
    assert (edges[:, 0] == edges[:, 1]).any() and len(np.unique(edges, axis=0)) < len(edges)
    return g, edges


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _rand(shape, seed, dtype=torch.float32, scale=1.0):
    g = torch.Generator("cuda").manual_seed(seed)
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


def _qkv(N, H, Dh, seed, dtype=torch.float32):
    return (_rand((N, H, Dh), seed, dtype, 1.0 / math.sqrt(Dh)), _rand((N, H, Dh), seed + 1, dtype),
            _rand((N, H, Dh), seed + 2, dtype))


def rel_err(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-12))


def restate(q, k, v, src, dst, n, mask=None, s=1.0):
    """The contract in torch, differentiable, in q's dtype: (out, lse); lse is -inf on empty rows."""
    sc = (q[dst] * k[src]).sum(-1)
    H = sc.shape[1]
    m = torch.full((n, H), -float("inf"), dtype=sc.dtype, device=sc.device)
    m = m.scatter_reduce(0, dst[:, None].expand(-1, H), sc, "amax")
    pe = torch.exp(sc - m[dst])
    l_ = torch.zeros((n, H), dtype=sc.dtype, device=sc.device).index_add(0, dst, pe)
    a = pe / l_[dst]
    beta = a if mask is None else a * mask * torch.tensor(s, dtype=sc.dtype, device=sc.device)
    out = torch.zeros_like(v).index_add(0, dst, v[src] * beta.unsqueeze(-1))
    return out, m + torch.log(l_)


def edge_mask(csr, H, p, seed=SEED):
    """[E, H] float32 keep mask in edge order from the library's host entry."""
    from pgl_b200 import _lib
    E = int(csr["cols"].shape[0])
    w = np.zeros(E, np.uint32)
    _lib.check(_lib.lib.pglb_attn_dropout_keep_host(seed[0], seed[1], p, 0, E, H, w.ctypes.data_as(ctypes.c_void_p)))
    bits = ((w[:, None] >> np.arange(H, dtype=np.uint32)) & 1).astype(np.float32)
    m = np.empty_like(bits)
    m[csr["eid"].cpu().numpy()] = bits
    return torch.from_numpy(m).cuda()


def _s32(p):
    return float(np.float32(1.0 / (1.0 - float(np.float32(p)))))


def fwd_raw(pgl, csr, q, k, v, drop=None):
    n, H, Dh = q.shape
    return pgl.ops._dot_attn_fwd_raw(csr, q.reshape(n, -1), k.reshape(n, -1), v.reshape(n, -1), H, Dh, drop, True)


def bwd_raw(pgl, csr, q, k, v, go, out, lse, drop=None):
    """The edge backward entry of q's dtype: (beta_e, ds_e) in edge order."""
    ops = pgl.ops
    n, H, Dh = q.shape
    q2, k2, v2, g2, o2 = (t.reshape(n, -1) for t in (q, k, v, go, out))
    E = int(csr["cols"].shape[0])
    beta = torch.empty((E, H), device="cuda")
    ds = torch.empty((E, H), device="cuda")
    dt = () if q.dtype == torch.float32 else (ops._DTYPE16[q.dtype],)
    name = "pglb_dot_attn_bwd_edge_%s%s" % ("drop_" if drop else "", "x16" if dt else "f32")
    ops.check(getattr(ops.lib, name)(
        ops._ptr(csr["rows"]), ops._ptr(csr["cols"]), ops._ptr(csr["eid"]), ops._ptr(q2), q2.stride(0), ops._ptr(k2),
        k2.stride(0), ops._ptr(v2), v2.stride(0), ops._ptr(g2), g2.stride(0), ops._ptr(o2), o2.stride(0), ops._ptr(lse),
        E, H, Dh, *dt, *(drop or ()), ops._ptr(beta), ops._ptr(ds), ops._stream()))
    return beta, ds


def _ends(edges):
    return torch.from_numpy(edges[:, 0]).cuda(), torch.from_numpy(edges[:, 1]).cuda()


@pytest.mark.parametrize("warm", ["0", "2"])   # launches before the checked one: each launch re-arms the task queue head
@pytest.mark.parametrize("H,Dh", LAYOUTS)
def test_forward_and_lse_against_float64(pgl, graph, warm, H, Dh):
    g, edges = graph
    N = g.num_nodes
    src, dst = _ends(edges)
    q, k, v = _qkv(N, H, Dh, 11 * H + Dh)
    first = [fwd_raw(pgl, g._fwd_csr(), q, k, v)[0] for _ in range(int(warm))]
    out, lse = fwd_raw(pgl, g._fwd_csr(), q, k, v)
    assert all(torch.equal(o, out) for o in first)
    want, wlse = restate(q.double(), k.double(), v.double(), src, dst, N)
    got = out.reshape(N, H, Dh)
    assert (got[-EMPTY:] == 0).all()
    assert float((got.double() - want).abs().max()) <= 1e-4 * float(want.abs().max())
    has = torch.isfinite(wlse)
    assert float((lse.double()[has] - wlse[has]).abs().max()) <= 1e-4 * max(1.0, float(wlse[has].abs().max()))
    assert (lse[~has] == 0).all()    # rows without in-edges are not written
    # inference (no lse) computes the same output bit for bit
    inf = pgl.ops.dot_attention(g._fwd_csr(), g._bwd_csr, q, k, v)
    assert torch.equal(_bits(inf), _bits(got))


@pytest.mark.parametrize("H,Dh", LAYOUTS)
def test_gradients_against_float64_autograd(pgl, graph, H, Dh):
    g, edges = graph
    N = g.num_nodes
    src, dst = _ends(edges)
    q, k, v = (t.requires_grad_() for t in _qkv(N, H, Dh, 23 * H + Dh))
    go = _rand((N, H, Dh), 5)
    out = pgl.ops.dot_attention(g._fwd_csr(), g._bwd_csr, q, k, v)
    got = torch.autograd.grad(out, (q, k, v), go)
    q64, k64, v64 = (t.detach().double().requires_grad_() for t in (q, k, v))
    want = torch.autograd.grad(restate(q64, k64, v64, src, dst, N)[0], (q64, k64, v64), go.double())
    for name, a, b in zip("qkv", got, want):
        assert a.dtype == torch.float32 and rel_err(a, b) <= GRAD_TOL, (name, rel_err(a, b))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 32), (2, 64), (8, 8), (16, 4), (32, 4)])
def test_x16_bit_exact_against_fp32_kernel(pgl, graph, dtype, H, Dh):
    g, edges = graph
    N = g.num_nodes
    fwd = g._fwd_csr()
    q, k, v = _qkv(N, H, Dh, 31 * H + Dh, dtype)
    out16, lse16 = fwd_raw(pgl, fwd, q, k, v)
    out32, lse32 = fwd_raw(pgl, fwd, q.float(), k.float(), v.float())
    assert out16.dtype == dtype
    assert torch.equal(_bits(out16), _bits(out32.to(dtype)))
    assert torch.equal(_bits(lse16), _bits(lse32))
    go = _rand((N, H, Dh), 7, dtype)
    o = out16.reshape(N, H, Dh)
    b16, d16 = bwd_raw(pgl, fwd, q, k, v, go, o, lse16)
    b32, d32 = bwd_raw(pgl, fwd, q.float(), k.float(), v.float(), go.float(), o.float(), lse16)
    assert torch.equal(_bits(b16), _bits(b32)) and torch.equal(_bits(d16), _bits(d32))


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 32), (16, 4)])
def test_x16_gradients_against_fp32_autograd(pgl, graph, dtype, H, Dh):
    """16-bit gradients: aggregated in fp32 and rounded once, with delta formed on the rounded output: within 4 u of
    the largest |grad| of fp32 torch autograd on the widened inputs."""
    g, edges = graph
    N = g.num_nodes
    src, dst = _ends(edges)
    q, k, v = (t.requires_grad_() for t in _qkv(N, H, Dh, 41 * H + Dh, dtype))
    go = _rand((N, H, Dh), 9, dtype)
    out = pgl.ops.dot_attention(g._fwd_csr(), g._bwd_csr, q, k, v)
    assert out.dtype == dtype
    got = torch.autograd.grad(out, (q, k, v), go)
    q32, k32, v32 = (t.detach().float().requires_grad_() for t in (q, k, v))
    want = torch.autograd.grad(restate(q32, k32, v32, src, dst, N)[0], (q32, k32, v32), go.float())
    for name, a, b in zip("qkv", got, want):
        assert a.dtype == dtype and rel_err(a, b) <= 4 * U[dtype], (name, rel_err(a, b))


@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 8), (32, 4)])
def test_dropout(pgl, graph, H, Dh):
    g, edges = graph
    N = g.num_nodes
    fwd = g._fwd_csr()
    src, dst = _ends(edges)
    p = 0.3
    drop = (p,) + SEED
    mask, s = edge_mask(fwd, H, p), _s32(p)
    assert 0.6 < float(mask.mean()) < 0.8
    q, k, v = _qkv(N, H, Dh, 51 * H + Dh)
    out, lse = fwd_raw(pgl, fwd, q, k, v, drop)
    out_again, _ = fwd_raw(pgl, fwd, q, k, v, drop)
    assert torch.equal(_bits(out), _bits(out_again))
    _, lse0 = fwd_raw(pgl, fwd, q, k, v)
    assert torch.equal(_bits(lse), _bits(lse0))              # lse is the value without dropout
    want, _ = restate(q, k, v, src, dst, N, mask, s)
    assert rel_err(out.reshape(N, H, Dh), want) <= 1e-4
    # the backward recomputes the same mask from (seed, offset): gradients against torch fp32 with that mask
    qg, kg, vg = (t.clone().requires_grad_() for t in (q, k, v))
    go = _rand((N, H, Dh), 13)
    o = pgl.ops.dot_attention(fwd, g._bwd_csr, qg, kg, vg, attn_drop=p, seed=SEED)
    assert torch.equal(_bits(o.detach().reshape(N, -1)), _bits(out))
    got = torch.autograd.grad(o, (qg, kg, vg), go)
    q2, k2, v2 = (t.clone().requires_grad_() for t in (q, k, v))
    want_g = torch.autograd.grad(restate(q2, k2, v2, src, dst, N, mask, s)[0], (q2, k2, v2), go)
    for name, a, b in zip("qkv", got, want_g):
        assert rel_err(a, b) <= GRAD_TOL, (name, rel_err(a, b))
    # 16-bit dropout forward: the fp32 one on the widened inputs, rounded
    for dtype in DTYPES:
        qh, kh, vh = (t.to(dtype) for t in (q, k, v))
        o16, l16 = fwd_raw(pgl, fwd, qh, kh, vh, drop)
        o32, l32 = fwd_raw(pgl, fwd, qh.float(), kh.float(), vh.float(), drop)
        assert torch.equal(_bits(o16), _bits(o32.to(dtype))) and torch.equal(_bits(l16), _bits(l32))


def test_calls_outside_the_kernels_return_none(pgl, graph):
    g, _ = graph
    N = g.num_nodes
    fwd, bwd = g._fwd_csr(), g._bwd_csr
    q, k, v = _qkv(N, 4, 8, 61)
    da = pgl.ops.dot_attention
    assert da(fwd, bwd, *_qkv(N, 4, 7, 62)) is None                        # head_dim 7 (concat=False citation layer)
    assert da(fwd, bwd, *_qkv(N, 4, 12, 63)) is None                       # head_dim not a power of two
    assert da(fwd, bwd, *_qkv(N, 16, 16, 64)) is None                      # 256 per row
    assert da(fwd, bwd, q, k, v.double()) is None and da(fwd, bwd, q.double(), k.double(), v.double()) is None
    assert da(fwd, bwd, q, k.half(), v) is None                            # dtype mix
    assert da(fwd, bwd, q[:-1], k[:-1], v[:-1]) is None                    # n_dst != N
    assert da(fwd, bwd, q, k, v, attn_drop=1.0) is None
    assert da(fwd, bwd, *_qkv(N, 2, 16, 65), attn_drop=0.5) is None        # dropout needs H % 4 == 0
    assert da({k_: v_ for k_, v_ in fwd.items() if k_ != "rows"}, bwd, q, k, v) is None
    assert da(fwd, bwd, *_qkv(N, 1, 4, 66, torch.bfloat16)) is None        # 8-byte 16-bit rows


def _op_by_op(conv, g, x):
    """TransformerConv.forward without edge features through the op-by-op route (send_uv, sum, edge_softmax,
    send_ue_recv), attn_drop = 0."""
    import pgl_b200.nn.functional as GF
    H, Dh = conv.num_heads, conv.hidden_size
    q = conv.q(x).reshape(-1, H, Dh) / (Dh ** 0.5)
    k = conv.k(x).reshape(-1, H, Dh)
    v = conv.v(x).reshape(-1, H, Dh)
    alpha = GF.edge_softmax(g, torch.sum(g.send_uv(k, q, "mul"), dim=-1)).reshape(-1, H, 1)
    out = g.send_ue_recv(v, alpha, "mul", "sum").reshape(-1, H * Dh)
    out = conv.layer_norm(conv.skip_feat(x) + out)
    return torch.relu(out)


def test_layer_gradients_and_launches_match_op_by_op(pgl, graph):
    g, _ = graph
    N = g.num_nodes
    torch.manual_seed(3)
    conv = pgl.nn.TransformerConv(32, 16, num_heads=8, feat_drop=0.0, attn_drop=0.0).cuda()
    x = _rand((N, 32), 71)
    go = _rand((N, 128), 72)
    params = list(conv.parameters())
    l0 = pgl.ops.launch_count()
    out = conv(g, x)
    got = torch.autograd.grad(out, params, go)
    torch.cuda.synchronize()
    l1 = pgl.ops.launch_count()
    ref = _op_by_op(conv, g, x)
    want = torch.autograd.grad(ref, params, go)
    torch.cuda.synchronize()
    l2 = pgl.ops.launch_count()
    assert rel_err(out, ref) <= 1e-4
    scale = max(float(b.abs().max()) for b in want)
    for (name, _), a, b in zip(conv.named_parameters(), got, want):
        if name == "k.bias":
            # k.bias shifts every score of a row by the same q . b, which the softmax removes: the exact gradient is 0
            # and both routes return rounding noise, bounded against the largest gradient of the layer
            assert float(a.abs().max()) <= 1e-4 * scale and float(b.abs().max()) <= 1e-4 * scale, name
            continue
        assert rel_err(a, b) <= 1e-4, (name, rel_err(a, b))
    assert l1 - l0 < l2 - l1, (l1 - l0, l2 - l1)
    with torch.no_grad():   # inference reaches the kernel without lse: the same output
        assert rel_err(conv.eval()(g, x), ref) <= 1e-4


def test_layer_peak_memory_has_no_edge_product(pgl):
    """E * H * Dh * 4 B (1 GB here) dwarfs everything else: the fused route's forward + backward peak stays well
    below the op-by-op route's and below one [E, H*Dh] tensor."""
    n, e = 20000, 2_000_000
    edges = O.chung_lu_edges(n, e, exponent=0.8, seed=81)
    g = pgl.Graph(edges=edges, num_nodes=n)
    g.tensor()
    conv = pgl.nn.TransformerConv(64, 16, num_heads=8, feat_drop=0.0, attn_drop=0.0).cuda()
    x = _rand((n, 64), 82)

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn(g, x).square().sum().backward()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    g._fwd_csr(), g._bwd_csr()
    fused = peak(conv)
    opby = peak(lambda gg, xx: _op_by_op(conv, gg, xx))
    edge_product = e * 128 * 4
    assert fused < edge_product and fused < 0.5 * opby, (fused, opby, edge_product)


def test_citation_model_trains_on_cora(pgl):
    """The reference citation benchmark's Transformer (2 x TransformerConv, 8 heads x 8, feat_drop = attn_drop = 0.6,
    Adam lr 0.005, weight decay 5e-4, 200 epochs).  The first layer runs the fused kernels with dropout; the second
    (concat=False, head_dim 7) stays op-by-op.  The reference publishes no figure for it: 0.75 is a sanity floor."""
    import torch.nn as nn
    c = O.load_cora(os.path.join(GOLDEN, "cora.npz"))
    n = c["num_nodes"]
    g = pgl.Graph(edges=c["edges"], num_nodes=n)
    g.tensor()
    x = torch.from_numpy(c["x"]).cuda()
    y = torch.from_numpy(c["y"]).cuda()
    idx = {k: torch.from_numpy(c[k + "_index"]).cuda() for k in ("train", "val", "test")}
    torch.manual_seed(0)
    T = pgl.nn.TransformerConv
    model = nn.ModuleList([T(1433, 8, 8, 0.6, 0.6, skip_feat=False, activation="relu"),
                           T(64, c["num_classes"], 8, 0.6, 0.6, concat=False, skip_feat=False, layer_norm=False,
                             activation=None)]).cuda()
    calls = []
    real = pgl.ops.dot_attention

    def counted(*a, **kw):
        r = real(*a, **kw)
        calls.append(r is not None)
        return r
    optim = torch.optim.Adam(model.parameters(), lr=0.005, weight_decay=5e-4)
    loss_fn = nn.CrossEntropyLoss()

    def fwd_model(inp):
        for m in model:
            inp = m(g, inp)
        return inp
    best_val, test_at_best = -1.0, 0.0
    pgl.ops.dot_attention = counted
    try:
        for epoch in range(200):
            model.train()
            loss = loss_fn(fwd_model(x)[idx["train"]], y[idx["train"]])
            optim.zero_grad()
            loss.backward()
            optim.step()
            model.eval()
            with torch.no_grad():
                pred = fwd_model(x).argmax(1)
            val = float((pred[idx["val"]] == y[idx["val"]]).float().mean())
            test = float((pred[idx["test"]] == y[idx["test"]]).float().mean())
            if val > best_val:
                best_val, test_at_best = val, test
    finally:
        pgl.ops.dot_attention = real
    assert any(calls) and not all(calls)     # layer 1 fused, layer 2 (head_dim 7) op-by-op
    print("transformer cora: best val %.3f, test at best val %.3f" % (best_val, test_at_best))
    assert test_at_best >= 0.75, (best_val, test_at_best)
