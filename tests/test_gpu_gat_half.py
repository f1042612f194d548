"""GATConv's fused aggregation and its backward on bfloat16 / float16 features (the *_x16 GAT entries).

Contract: features are widened exactly; logits, softmax, rescales and accumulation run in fp32 with the fp32 kernels'
instructions and slot order; each 16-bit output is rounded once.  So the forward output is round16(the fp32 kernel on
the widened features) bit for bit, lse / alpha_e / dz_e / the attention projections equal the fp32 kernels' on the
widened inputs bit for bit, and grad f (a reverse-CSR sum formed in fp32) is within 2 u |ref32|_inf of the fp32
library (u = 2^-8 bf16, 2^-11 fp16)."""

import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
DTYPES = (torch.bfloat16, torch.float16)
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
EMPTY = 64   # trailing nodes without an edge: empty rows


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


@pytest.fixture(scope="module")
def graph(pgl):
    """Rows cut across tasks (in-degree > 2048), one-edge rows and empty rows."""
    n = 3000
    edges = O.chung_lu_edges(n, 80000, exponent=0.9, seed=301)
    g = pgl.Graph(edges=edges, num_nodes=n + EMPTY)
    g.tensor()
    deg = np.bincount(edges[:, 1], minlength=n + EMPTY)
    assert deg.max() > 2048 and (deg == 0).sum() >= EMPTY and (deg == 1).sum() > 0
    return g, edges


def _bits(t):
    return t.contiguous().view(torch.int16)


def _rand(shape, seed, dtype=torch.float32):
    return torch.randn(shape, device="cuda", generator=torch.Generator("cuda").manual_seed(seed)).to(dtype)


def _normwise(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / b.norm())


def torch_gat(f, a_s, a_d, src, dst, n, slope):
    """out[d,h,:] = sum_j softmax_j(leaky(a_s[src_j,h] + a_d[d,h])) f[src_j,h,:] in plain torch (differentiable)."""
    z = torch.nn.functional.leaky_relu(a_s[src] + a_d[dst], slope)
    H = z.shape[1]
    m = torch.full((n, H), -float("inf"), device=z.device).scatter_reduce(0, dst[:, None].expand(-1, H), z, "amax")
    p = torch.exp(z - m[dst])
    s = torch.zeros((n, H), device=z.device).index_add(0, dst, p)
    al = p / s[dst]
    return torch.zeros_like(f).index_add(0, dst, f[src] * al.unsqueeze(-1)), al


def _fused_raw(pgl, csr, f2, a_s, a_d, slope, H, Dh):
    """The train entry of f2's dtype: (out [n_dst, H*Dh] in f2's dtype, lse [n_dst, H] float32)."""
    from pgl_b200 import ops
    lib = ops.lib
    n_src = int(f2.shape[0])
    E = int(csr["cols"].shape[0])
    n_dst = int(csr["indptr"].shape[0]) - 1
    out = torch.empty((n_dst, H * Dh), dtype=f2.dtype, device="cuda")
    lse = torch.zeros((n_dst, H), dtype=torch.float32, device="cuda")
    ws = ops.workspace(f2.device, 1 << 28)
    args = (ops._ptr(csr["indptr"]), ops._ptr(csr["cols"]), ops._ptr(f2), f2.stride(0), ops._ptr(a_s), ops._ptr(a_d),
            float(slope), ops._ptr(out), out.stride(0), ops._ptr(lse), n_dst, n_src, E, H, Dh)
    if f2.dtype == torch.float32:
        ops.check(lib.pglb_gat_fused_train_csr_f32(*args, ops._ptr(ws), ws.numel(), ops._stream()))
    else:
        ops.check(lib.pglb_gat_fused_train_csr_x16(*args, ops._DTYPE16[f2.dtype], ops._ptr(ws), ws.numel(),
                                                   ops._stream()))
    return out, lse


# 1. forward, bit-exact -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 32), (16, 8), (12, 8)])
@pytest.mark.parametrize("slope", [0.2, 0.0, 1.0])
def test_forward_is_round16_of_fp32(pgl, graph, dtype, H, Dh, slope):
    g, _ = graph
    ops = pgl.ops
    csr = g._fwd_csr()
    N = int(g.num_nodes)
    f = _rand((N, H, Dh), 401 + H, dtype)
    a_s, a_d = _rand((N, H), 402), _rand((N, H), 403)
    with torch.no_grad():
        want = ops.gat_fused(csr, f.float(), a_s, a_d, slope)
        got = ops.gat_fused(csr, f, a_s, a_d, slope, out_dtype=dtype)
    assert got.dtype == dtype and torch.equal(_bits(got), _bits(want.to(dtype)))
    out32, lse32 = _fused_raw(pgl, csr, f.float().reshape(N, -1), a_s, a_d, slope, H, Dh)
    out16, lse16 = _fused_raw(pgl, csr, f.reshape(N, -1), a_s, a_d, slope, H, Dh)
    assert torch.equal(_bits(out16), _bits(out32.to(dtype)))
    assert torch.equal(lse16.view(torch.int32), lse32.view(torch.int32))
    tr = ops.gat_fused_train(csr, g._bwd_csr, f, a_s, a_d, slope, out_dtype=dtype)
    assert tr is not None and torch.equal(_bits(tr), _bits(want.to(dtype)))
    # the default result dtype is unchanged: torch promotion (bf16 features with fp32 attention give fp32)
    with torch.no_grad():
        assert torch.equal(ops.gat_fused(csr, f, a_s, a_d, slope), want)
        both16 = ops.gat_fused(csr, f, a_s.to(dtype), a_d.to(dtype), slope)
        assert both16.dtype == dtype
        assert torch.equal(_bits(both16), _bits(ops.gat_fused(csr, f.float(), a_s.to(dtype).float(),
                                                              a_d.to(dtype).float(), slope).to(dtype)))


# 2. edge backward, bit-exact -----------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 32), (16, 8)])
def test_edge_backward_is_the_fp32_kernel_on_widened_inputs(pgl, graph, dtype, H, Dh):
    g, _ = graph
    ops = pgl.ops
    fwd = g._fwd_csr()
    N = int(g.num_nodes)
    E = int(fwd["cols"].shape[0])
    f = _rand((N, H * Dh), 411, dtype)
    go = _rand((N, H * Dh), 412, dtype)
    a_s, a_d = _rand((N, H), 413), _rand((N, H), 414)
    out16, lse = _fused_raw(pgl, fwd, f, a_s, a_d, 0.2, H, Dh)
    res = {}
    for name, (ff, gg, oo) in (("x16", (f, go, out16)), ("f32", (f.float(), go.float(), out16.float()))):
        alpha = torch.empty((E, H), device="cuda")
        dz = torch.empty((E, H), device="cuda")
        args = [ops._ptr(fwd["rows"]), ops._ptr(fwd["cols"]), ops._ptr(fwd["eid"]), ops._ptr(ff), ff.stride(0),
                ops._ptr(gg), gg.stride(0), ops._ptr(oo), oo.stride(0), ops._ptr(a_s), ops._ptr(a_d), ops._ptr(lse),
                0.2, E, H, Dh]
        if name == "x16":
            ops.check(ops.lib.pglb_gat_bwd_edge_x16(*args, ops._DTYPE16[dtype], ops._ptr(alpha), ops._ptr(dz),
                                                    ops._stream()))
        else:
            ops.check(ops.lib.pglb_gat_bwd_edge_f32(*args, ops._ptr(alpha), ops._ptr(dz), ops._stream()))
        res[name] = (alpha, dz)
    for a, b in zip(res["x16"], res["f32"]):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


# 3. the reverse aggregation with an edge operand ---------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
def test_spmm_ue_x16_bar_and_determinism(pgl, graph, dtype):
    from pgl_b200._lib import BCAST_HEAD, BCAST_SCALAR
    g, _ = graph
    ops = pgl.ops
    bwd = g._bwd_csr()
    N = int(g.num_nodes)
    E = int(bwd["cols"].shape[0])
    for D, H, bcast, msg in ((128, 8, BCAST_HEAD, "mul"), (96, 12, BCAST_HEAD, "add"), (128, 1, BCAST_SCALAR, "mul"),
                             (64, 1, BCAST_SCALAR, "add")):
        x = _rand((N, D), 421 + D, dtype)
        y = torch.rand((E, H), device="cuda", generator=torch.Generator("cuda").manual_seed(422 + H))
        kw = dict(eid=bwd["eid"], y2=y, y_bcast=bcast, head_dim=D // H if bcast == BCAST_HEAD else 1, msg_op=msg)
        for hint in (-1, bwd.get("max_degree", -1)):   # hub passes on and as the graph's own hint decides
            got = ops._spmm_raw(bwd["indptr"], bwd["cols"], x, N, "sum", max_degree=hint, **kw)
            again = ops._spmm_raw(bwd["indptr"], bwd["cols"], x, N, "sum", max_degree=hint, **kw)
            ref = ops._spmm_raw(bwd["indptr"], bwd["cols"], x.float(), N, "sum", max_degree=hint, **kw)
            assert got.dtype == dtype and torch.equal(_bits(got), _bits(again)), (D, msg)
            err = float((got.double() - ref.double()).abs().max())
            assert err <= 2 * U[dtype] * float(ref.abs().max()), (D, msg, err)


# 4. gradients ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 32), (32, 4)])
def test_gradients_against_torch_fp32(pgl, graph, dtype, H, Dh):
    """Bars (normwise, against plain torch fp32 autograd on the widened inputs): 2 u for the output and for grad f
    (each is a fp32 result rounded once), 16 u of the largest grad attn_src entry for the attention gradients (the
    backward's delta = <grad_out, out> uses the rounded 16-bit out; with slope 1 grad attn_dst cancels to 0 exactly)."""
    g, edges = graph
    N = int(g.num_nodes)
    src = torch.from_numpy(edges[:, 0]).cuda()
    dst = torch.from_numpy(edges[:, 1]).cuda()
    f1 = _rand((N, H, Dh), 431, dtype).requires_grad_(True)
    s1 = _rand((N, H), 432).requires_grad_(True)
    d1 = _rand((N, H), 433, dtype).requires_grad_(True)   # attention of either dtype: gradients come back in it
    go = _rand((N, H, Dh), 434, dtype)
    out = pgl.ops.gat_fused_train(g._fwd_csr(), g._bwd_csr, f1, s1, d1, 0.2, out_dtype=dtype)
    assert out is not None and out.dtype == dtype
    out.backward(go)
    assert f1.grad.dtype == dtype and s1.grad.dtype == torch.float32 and d1.grad.dtype == dtype
    f2, s2, d2 = [t.detach().float().requires_grad_(True) for t in (f1, s1, d1)]
    ref, _ = torch_gat(f2, s2, d2, src, dst, N, 0.2)
    ref.backward(go.float())
    assert _normwise(out, ref) <= 2 * U[dtype]
    assert _normwise(f1.grad, f2.grad) <= 2 * U[dtype]
    scale = float(s2.grad.abs().max())
    assert float((s1.grad - s2.grad).abs().max()) <= 16 * U[dtype] * scale
    # grad attn_dst is rounded to its dtype once: half an ulp of its own size on top
    tol_d = 16 * U[dtype] * max(scale, float(d2.grad.abs().max()))
    assert float((d1.grad.float() - d2.grad).abs().max()) <= tol_d


# 5. attention projections ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 8), (1, 128), (32, 4), (12, 8)])
def test_head_dots_is_the_fp32_kernel_on_widened_inputs(pgl, dtype, H, Dh):
    n = 5003
    f = _rand((n, H, Dh), 441 + H, dtype)
    ws, wd = _rand((H, Dh), 442), _rand((H, Dh), 443)
    for w_s, w_d in ((ws, wd), (ws.to(dtype), wd.to(dtype))):
        got = pgl.ops.head_dots(f, w_s, w_d)
        want = pgl.ops.head_dots(f.float(), w_s.float(), w_d.float())
        assert got is not None and got[0].dtype == torch.float32
        for a, b in zip(got, want):
            assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    # gradients come back in each input's dtype
    f1 = f.clone().requires_grad_(True)
    w1, w2 = ws.clone().requires_grad_(True), wd.to(dtype).requires_grad_(True)
    a_s, a_d = pgl.ops.head_dots(f1, w1, w2)
    (a_s.sum() + 2 * a_d.sum()).backward()
    assert f1.grad.dtype == dtype and w1.grad.dtype == torch.float32 and w2.grad.dtype == dtype
    f2, v1, v2 = f.float().requires_grad_(True), ws.clone().requires_grad_(True), wd.to(dtype).float().requires_grad_(True)
    (torch.sum(f2 * v1, -1).sum() + 2 * torch.sum(f2 * v2, -1).sum()).backward()
    assert _normwise(f1.grad, f2.grad) <= U[dtype]
    assert _normwise(w1.grad, v1.grad) <= 1e-5 and _normwise(w2.grad, v2.grad) <= U[dtype]


@pytest.mark.parametrize("dtype", DTYPES)
def test_head_dots_declines_what_the_kernel_cannot_read(pgl, dtype):
    """16-bit rows of H*Dh % 8 != 0 elements are not a multiple of 16 bytes, and float32 weights reach the kernel
    uncopied: both give None (the caller keeps the torch expressions), never a library error."""
    for H, Dh in ((3, 4), (1, 4), (5, 4)):
        f = _rand((100, H, Dh), 451, dtype)
        assert pgl.ops.head_dots(f, _rand((H, Dh), 452), _rand((H, Dh), 453)) is None
        assert pgl.ops.head_dots(f.float(), _rand((H, Dh), 452), _rand((H, Dh), 453)) is not None   # fp32: 16-byte rows
    f = _rand((100, 8, 16), 454, dtype)
    buf = _rand((8 * 16 + 1,), 455)
    w_mis = buf[1:].reshape(8, 16)   # contiguous, 4 bytes past a 16-byte boundary
    assert w_mis.is_contiguous() and w_mis.data_ptr() % 16
    assert pgl.ops.head_dots(f, w_mis, _rand((8, 16), 456)) is None
    assert pgl.ops.head_dots(f, w_mis.to(dtype), _rand((8, 16), 456)) is not None   # 16-bit weights are copied


@pytest.mark.parametrize("dtype", DTYPES)
def test_32_heads_x_4(pgl, graph, dtype):
    """32 heads x 4 fit the 16-bit rings but not the fp32 ones, so no fp32 output is bitwise comparable: the 16-bit
    output is within 2 u |ref32|_inf of the fp32 inference entry (its per-slot kernel) on the widened features, and lse
    within 1e-4 (relative) of the log-sum-exp computed in float64."""
    g, edges = graph
    ops = pgl.ops
    csr = g._fwd_csr()
    N, H, Dh = int(g.num_nodes), 32, 4
    f = _rand((N, H, Dh), 461, dtype)
    a_s, a_d = _rand((N, H), 462), _rand((N, H), 463)
    with torch.no_grad():
        ref = ops.gat_fused(csr, f.float(), a_s, a_d, 0.2)
        got = ops.gat_fused(csr, f, a_s, a_d, 0.2, out_dtype=dtype)
    assert got.dtype == dtype
    assert float((got.double() - ref.double()).abs().max()) <= 2 * U[dtype] * float(ref.abs().max())
    out16, lse = _fused_raw(pgl, csr, f.reshape(N, -1), a_s, a_d, 0.2, H, Dh)
    assert torch.equal(_bits(out16), _bits(got.reshape(N, -1)))
    src = torch.from_numpy(edges[:, 0]).cuda()
    dst = torch.from_numpy(edges[:, 1]).cuda()
    z = torch.nn.functional.leaky_relu(a_s.double()[src] + a_d.double()[dst], 0.2)
    m = torch.full((N, H), -float("inf"), device="cuda", dtype=torch.float64).scatter_reduce(
        0, dst[:, None].expand(-1, H), z, "amax")
    s = torch.zeros((N, H), device="cuda", dtype=torch.float64).index_add(0, dst, torch.exp(z - m[dst]))
    has = torch.bincount(dst, minlength=N) > 0
    want = (m + torch.log(s))[has]
    assert float((lse.double()[has] - want).abs().max()) <= 1e-4 * max(1.0, float(want.abs().max()))
    # the fp32 train entry refuses this shape (the layer stays op-by-op in fp32)
    with pytest.raises(pgl._lib.PglbError):
        _fused_raw(pgl, csr, f.float().reshape(N, -1), a_s, a_d, 0.2, H, Dh)


# 6. the layer ------------------------------------------------------------------------------------------------------
X16_ENTRIES = ("pglb_gat_fused_csr_x16", "pglb_gat_fused_train_csr_x16", "pglb_gat_bwd_edge_x16",
               "pglb_spmm_csr_ue_x16", "pglb_head_dots_x16")


def _spy(monkeypatch, ops):
    calls = {k: 0 for k in X16_ENTRIES}
    for name in X16_ENTRIES:
        real = getattr(ops.lib, name)

        def spy(*a, _real=real, _name=name):
            calls[_name] += 1
            return _real(*a)
        monkeypatch.setattr(ops.lib, name, spy)
    return calls


def test_gatconv_bf16_takes_the_fused_path(pgl, graph, monkeypatch):
    g, _ = graph
    ops = pgl.ops
    N = int(g.num_nodes)
    torch.manual_seed(0)
    ref_layer = pgl.nn.GATConv(96, 16, feat_drop=0.0, attn_drop=0.0, num_heads=8).cuda()
    x = torch.randn(N, 96, device="cuda")
    x32 = x.clone().requires_grad_()
    ref = ref_layer(g, x32)
    ref.backward(torch.ones_like(ref))
    layer = pgl.nn.GATConv(96, 16, feat_drop=0.0, attn_drop=0.0, num_heads=8).cuda()
    layer.load_state_dict(ref_layer.state_dict())
    layer = layer.to(torch.bfloat16)
    g._fwd_csr(), g._bwd_csr()   # the one-off index builds are not part of a layer's launch count

    def run(fused):
        old = ops.GAT_FUSED_TRAIN
        ops.GAT_FUSED_TRAIN = fused
        try:
            layer.zero_grad()
            x16 = x.to(torch.bfloat16).requires_grad_()
            l0 = ops.launch_count()
            out = layer(g, x16)
            fwd_launches = ops.launch_count() - l0
            out.backward(torch.ones_like(out))
            return out.detach(), x16.grad, fwd_launches
        finally:
            ops.GAT_FUSED_TRAIN = old

    calls = _spy(monkeypatch, ops)
    out_f, gx_f, n_f = run(True)
    assert calls["pglb_gat_fused_train_csr_x16"] == 1 and calls["pglb_gat_bwd_edge_x16"] == 1
    assert calls["pglb_spmm_csr_ue_x16"] == 1 and calls["pglb_head_dots_x16"] == 1
    out_u, gx_u, n_u = run(False)
    assert n_f < n_u
    for out, gx in ((out_f, gx_f), (out_u, gx_u)):
        assert out.dtype == torch.bfloat16 and gx.dtype == torch.bfloat16
        assert _normwise(out, ref) <= 3e-2 and _normwise(gx, x32.grad) <= 3e-2
    for p in layer.parameters():
        assert p.grad.dtype == torch.bfloat16
    layer.eval()
    with torch.no_grad():
        out_e = layer(g, x.to(torch.bfloat16))
    assert calls["pglb_gat_fused_csr_x16"] == 1
    assert out_e.dtype == torch.bfloat16 and _normwise(out_e, ref) <= 3e-2


@pytest.mark.parametrize("H,Dh,attn_drop", [(3, 32, 0.0), (32, 4, 0.0), (5, 12, 0.0), (4, 24, 0.0), (8, 16, 0.5),
                                                (3, 4, 0.0), (1, 4, 0.0)])
def test_gatconv_bf16_other_shapes_keep_their_dtypes(pgl, graph, H, Dh, attn_drop):
    """H % 4 != 0, 32 heads, D % 8 != 0 (also with head_dim 4, where the 16-bit projections fall back to the torch
    expressions), a head_dim that is not a power of two and attention dropout: whichever path
    runs, a bf16 layer gives bf16 outputs and gradients, and an fp32 layer under bf16 autocast gives fp32 outputs."""
    g, _ = graph
    N = int(g.num_nodes)
    torch.manual_seed(1)
    layer = pgl.nn.GATConv(40, Dh, feat_drop=0.0, attn_drop=attn_drop, num_heads=H).cuda()
    x = torch.randn(N, 40, device="cuda")
    l16 = pgl.nn.GATConv(40, Dh, feat_drop=0.0, attn_drop=attn_drop, num_heads=H).cuda()
    l16.load_state_dict(layer.state_dict())
    l16 = l16.to(torch.bfloat16).train()
    x16 = x.to(torch.bfloat16).requires_grad_()
    out = l16(g, x16)
    assert out.dtype == torch.bfloat16
    out.backward(torch.ones_like(out))
    assert x16.grad.dtype == torch.bfloat16 and torch.isfinite(x16.grad.float()).all()
    for p in l16.parameters():
        assert p.grad.dtype == torch.bfloat16
    l16.eval()
    with torch.no_grad():
        assert l16(g, x.to(torch.bfloat16)).dtype == torch.bfloat16
    xa = x.clone().requires_grad_()
    with torch.autocast("cuda", dtype=torch.bfloat16):
        out_a = layer(g, xa)
    assert out_a.dtype == torch.float32
    out_a.backward(torch.ones_like(out_a))
    assert xa.grad.dtype == torch.float32


def test_bf16_training_tracks_fp32(pgl, graph):
    """GATConv(32 -> 8 x 16) + a linear classifier (fused training path, attn_drop = 0) on a synthetic task whose label
    is a linear function of the in-neighbours' features: 40 Adam steps from one init in fp32 and as a bf16 module.  The
    bf16 loss stays within 0.05 + 5 % of the fp32 loss at every step, and both runs learn."""
    g, _ = graph
    N = int(g.num_nodes)
    nn = pgl.nn
    gen = torch.Generator("cuda").manual_seed(451)
    x = torch.randn(N, 32, device="cuda", generator=gen)
    teacher = torch.randn(32, 6, device="cuda", generator=gen)
    with torch.no_grad():
        y = g.send_recv(x @ teacher, "mean").argmax(-1)

    class Net(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.c1 = nn.GATConv(32, 16, feat_drop=0.0, attn_drop=0.0, num_heads=8)
            self.out = torch.nn.Linear(128, 6)

        def forward(self, h):
            return self.out(self.c1(g, h))

    torch.manual_seed(2)
    net32 = Net().cuda()
    net16 = Net().cuda()
    net16.load_state_dict(net32.state_dict())
    net16 = net16.to(torch.bfloat16)
    losses = {}
    for name, net, xin in (("fp32", net32, x), ("bf16", net16, x.to(torch.bfloat16))):
        opt = torch.optim.Adam(net.parameters(), lr=1e-2)
        ls = []
        for _ in range(40):
            opt.zero_grad()
            loss = torch.nn.functional.cross_entropy(net(xin).float(), y)
            loss.backward()
            opt.step()
            ls.append(float(loss.detach()))
        losses[name] = ls
    a, b = np.array(losses["fp32"]), np.array(losses["bf16"])
    assert np.all(np.abs(b - a) <= 0.05 + 0.05 * a), (a, b)
    assert a[-1] < 0.7 * a[0] and b[-1] < 0.7 * b[0]
