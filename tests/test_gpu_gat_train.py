"""Fused GAT under autograd (pglb_gat_fused_train_csr_f32 + pglb_gat_bwd_edge_f32) and the device-side task queue of
the persistent kernels: forward against the oracle restatement of pgl/nn/conv.py:308-346, every gradient against plain
torch fp32 autograd of the same formula."""
import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
RTOL = 1e-4


def rel_err(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-12) if a.size else 0.0


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def make_graph(pgl, edges, n):
    g = pgl.Graph(edges=np.asarray(edges, np.int64), num_nodes=n)
    g.tensor()
    return g


def torch_gat(f, a_s, a_d, src, dst, n, slope):
    """out[d,h,:] = sum_j softmax_j(leaky(a_s[src_j,h] + a_d[d,h])) f[src_j,h,:] in plain torch (differentiable)."""
    z = torch.nn.functional.leaky_relu(a_s[src] + a_d[dst], slope)
    H = z.shape[1]
    m = torch.full((n, H), -float("inf"), device=z.device).scatter_reduce(0, dst[:, None].expand(-1, H), z, "amax")
    p = torch.exp(z - m[dst])
    s = torch.zeros((n, H), device=z.device).index_add(0, dst, p)
    al = p / s[dst]
    return torch.zeros_like(f).index_add(0, dst, f[src] * al.unsqueeze(-1)), al


@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 32), (16, 8), (12, 8)])
@pytest.mark.parametrize("slope", [0.2, 0.0, 1.0])
def test_gat_fused_train_forward_and_gradients(pgl, H, Dh, slope):
    """Hubs (rows cut across tasks: lse comes from the merge kernel), empty rows, one-edge rows."""
    n, e = 3000, 80000
    edges = O.chung_lu_edges(n, e, exponent=0.9, seed=301)
    g = make_graph(pgl, edges, n)
    assert g.adj_dst_index.max_degree > 2048
    src, dst = dev(edges[:, 0]), dev(edges[:, 1])
    gen = torch.Generator(device="cuda").manual_seed(302)
    f1 = torch.randn(n, H, Dh, device="cuda", generator=gen).requires_grad_(True)
    s1 = torch.randn(n, H, device="cuda", generator=gen).requires_grad_(True)
    d1 = torch.randn(n, H, device="cuda", generator=gen).requires_grad_(True)
    go = torch.randn(n, H, Dh, device="cuda", generator=gen)
    out = pgl.ops.gat_fused_train(g._fwd_csr(), g._bwd_csr, f1, s1, d1, slope)
    assert out is not None and out.shape == (n, H, Dh)
    out.backward(go)
    f2, s2, d2 = [t.detach().clone().requires_grad_(True) for t in (f1, s1, d1)]
    ref, _ = torch_gat(f2, s2, d2, src, dst, n, slope)
    ref.backward(go)
    assert rel_err(out.detach().cpu().numpy(), ref.detach().cpu().numpy()) <= RTOL, "forward"
    assert rel_err(f1.grad.cpu().numpy(), f2.grad.cpu().numpy()) <= RTOL, "grad f"
    # the logit gradients are differences of O(|go| |f|) terms (d alpha - <go, out>); with slope = 1 the row sums that
    # make grad attn_dst cancel to exactly 0 in exact arithmetic: judge both against the size of grad attn_src
    scale = float(s2.grad.abs().max())
    assert float((s1.grad - s2.grad).abs().max()) <= 5e-4 * scale, "grad attn_src"
    assert float((d1.grad - d2.grad).abs().max()) <= 5e-4 * max(scale, float(d2.grad.abs().max())), "grad attn_dst"
    # the forward is the inference kernel: same numbers with autograd off
    with torch.no_grad():
        inf = pgl.ops.gat_fused(g._fwd_csr(), f1.detach(), s1.detach(), d1.detach(), slope)
    assert torch.equal(inf, out.detach())


def test_gat_fused_train_pieces_against_oracle(pgl):
    """alpha_e rebuilt by the backward edge kernel == the oracle's edge_softmax(leaky(send_uv)) in edge order."""
    n, e, H, Dh = 2000, 30000, 8, 16
    edges = O.chung_lu_edges(n, e, exponent=0.8, seed=311)
    g = make_graph(pgl, edges, n)
    rng = np.random.default_rng(312)
    f = rng.standard_normal((n, H, Dh)).astype(np.float32)
    a_s = rng.standard_normal((n, H)).astype(np.float32)
    a_d = rng.standard_normal((n, H)).astype(np.float32)
    ft = dev(f).requires_grad_(True)
    out = pgl.ops.gat_fused_train(g._fwd_csr(), g._bwd_csr, ft, dev(a_s), dev(a_d), 0.2)
    # gradient of sum(out * f_const) wrt f: alpha-weighted reverse aggregation; compare its ingredients
    al = O.send_uv(a_s, a_d, edges[:, 0], edges[:, 1], "add")
    al = np.where(al >= 0, al, al * np.float32(0.2)).astype(np.float32)
    al = O.edge_softmax(edges, n, al, "dst")
    want = O.send_ue_recv(f.reshape(n, H, Dh), al.reshape(-1, H, 1), edges[:, 0], edges[:, 1], "mul", "sum")
    assert rel_err(out.detach().cpu().numpy(), want) <= RTOL
    go = rng.standard_normal((n, H, Dh)).astype(np.float32)
    out.backward(dev(go))
    # grad f[s] = sum_{e: src=s} alpha[e] * go[dst[e]]  -> the oracle's send_ue_recv on the reversed edges
    rev = np.ascontiguousarray(edges[:, ::-1])
    want_gf = O.send_ue_recv(go, al.reshape(-1, H, 1), rev[:, 0], rev[:, 1], "mul", "sum")
    assert rel_err(ft.grad.cpu().numpy(), want_gf) <= RTOL


def test_gat_conv_trains_on_the_fused_path(pgl):
    """GATConv(8 x 16) forward + backward: fused training path vs op-by-op path vs plain torch."""
    n, e, H, Dh, fin = 1500, 30000, 8, 16, 24
    edges = O.chung_lu_edges(n, e, exponent=0.8, seed=321)
    g = make_graph(pgl, edges, n)
    src, dst = dev(edges[:, 0]), dev(edges[:, 1])
    torch.manual_seed(5)
    conv = pgl.nn.GATConv(fin, Dh, feat_drop=0, attn_drop=0, num_heads=H, concat=True).cuda()
    x0 = torch.randn(n, fin, device="cuda")
    go = torch.randn(n, H * Dh, device="cuda")
    g._fwd_csr(), g._bwd_csr()   # the one-off index builds are not part of a layer's launch count

    def run(fused):
        old = pgl.ops.GAT_FUSED_TRAIN
        pgl.ops.GAT_FUSED_TRAIN = fused
        try:
            conv.zero_grad()
            x = x0.clone().requires_grad_(True)
            l0 = pgl.ops.launch_count()
            out = conv(g, x)
            fwd_launches = pgl.ops.launch_count() - l0
            out.backward(go)
            return out.detach(), x.grad.clone(), {k: p.grad.clone() for k, p in conv.named_parameters()}, fwd_launches
        finally:
            pgl.ops.GAT_FUSED_TRAIN = old

    out_f, gx_f, gp_f, nf = run(True)
    out_u, gx_u, gp_u, nu = run(False)
    assert nf < nu  # one aggregation launch (+ plan / empty rows / merge) instead of send_uv + softmax + send_ue_recv
    conv.zero_grad()
    x2 = x0.clone().requires_grad_(True)
    f = (x2 @ conv.linear.weight + conv.linear.bias).reshape(-1, H, Dh)
    ref, _ = torch_gat(f, (f * conv.weight_src).sum(-1), (f * conv.weight_dst).sum(-1), src, dst, n, 0.2)
    ref = ref.reshape(n, H * Dh)
    ref.backward(go)
    for got_out, got_gx, got_gp in ((out_f, gx_f, gp_f), (out_u, gx_u, gp_u)):
        assert rel_err(got_out.cpu().numpy(), ref.detach().cpu().numpy()) <= RTOL
        assert rel_err(got_gx.cpu().numpy(), x2.grad.cpu().numpy()) <= 5e-4
        for k, p in conv.named_parameters():
            assert rel_err(got_gp[k].cpu().numpy(), p.grad.cpu().numpy()) <= 5e-4, k
    # attention dropout in training mode keeps the op-by-op path (dropout acts on alpha)
    conv2 = pgl.nn.GATConv(fin, Dh, feat_drop=0, attn_drop=0.5, num_heads=H).cuda().train()
    y = conv2(g, x0.clone().requires_grad_(True))
    y.sum().backward()
    assert torch.isfinite(y).all()


def test_gat_fused_train_unsupported_shapes_fall_back(pgl):
    n, e = 500, 4000
    edges = O.chung_lu_edges(n, e, exponent=0.7, seed=331)
    g = make_graph(pgl, edges, n)
    # narrow row, H % 4, H % 4, head_dim not a power of two, 32 heads (attention rows too wide for the kernel's rings)
    for H, Dh in ((4, 8), (3, 32), (2, 64), (8, 12), (32, 4)):
        f = torch.randn(n, H, Dh, device="cuda", requires_grad=True)
        a = torch.randn(n, H, device="cuda")
        assert pgl.ops.gat_fused_train(g._fwd_csr(), g._bwd_csr, f, a, a, 0.2) is None
    f = torch.randn(n, 8, 16, device="cuda", requires_grad=True)
    a = torch.randn(n, 8, device="cuda")
    assert pgl.ops.gat_fused_train(g._fwd_csr(), g._bwd_csr, f, a, a, 1.5) is None   # slope outside [0, 1]
    # 32 heads x 4 at inference: outside the TMA kernel's shared-memory budget -> round 1's single-pass kernel
    src, dst = dev(edges[:, 0]), dev(edges[:, 1])
    f32 = torch.randn(n, 32, 4, device="cuda")
    a32, b32 = torch.randn(n, 32, device="cuda"), torch.randn(n, 32, device="cuda")
    with torch.no_grad():
        got = pgl.ops.gat_fused(g._fwd_csr(), f32, a32, b32, 0.2)
        ref, _ = torch_gat(f32, a32, b32, src, dst, n, 0.2)
    assert got is not None and rel_err(got.cpu().numpy(), ref.cpu().numpy()) <= RTOL
    # the layers still train on those shapes (op-by-op path)
    conv = pgl.nn.GATConv(10, 8, feat_drop=0, attn_drop=0, num_heads=4).cuda()
    x = torch.randn(n, 10, device="cuda", requires_grad=True)
    conv(g, x).sum().backward()
    assert torch.isfinite(x.grad).all()


# ---------------------------------------------------------------- device-side task queue
@pytest.mark.parametrize("order", [1, 2])
def test_dynamic_task_queue_is_bit_identical(pgl, order):
    """Which warp runs a task does not enter the arithmetic, and every launch's plan kernel re-arms the queue head that
    the copy-sum and GAT kernels share through the workspace: repeat launches give the same bits, copy-sum and GAT
    alike (hub rows cut into task partials included: the merge kernels add them in task order).  order 1: each call
    repeated back to back; 2: the calls interleaved."""
    n, e, d = 6000, 200000, 128
    edges = O.chung_lu_edges(n, e, exponent=0.9, seed=341)
    g = make_graph(pgl, edges, n)
    gen = torch.Generator(device="cuda").manual_seed(342)
    x = torch.randn(n, d, device="cuda", generator=gen)
    norm = torch.rand(n, device="cuda", generator=gen) + 0.5
    a_s = torch.randn(n, 8, device="cuda", generator=gen)
    a_d = torch.randn(n, 8, device="cuda", generator=gen)
    calls = [lambda: g._send_u_recv(x, "sum", None),
             lambda: g._send_u_recv(x, "sum", None, scale_src=norm, scale_dst=norm),
             lambda: g._send_u_recv(x[:, :100].contiguous(), "mean", None),
             lambda: pgl.ops.gat_fused(g._fwd_csr(), x.reshape(n, 8, 16), a_s, a_d, 0.2)]
    with torch.no_grad():
        base = [c() for c in calls]
        seq = [i for i in range(len(calls)) for _ in range(3)] if order == 1 else list(range(len(calls))) * 3
        for i in seq:
            assert torch.equal(calls[i](), base[i]), i
    base_sum = base[0]
    want = O.send_u_recv(x.cpu().numpy(), edges[:, 0], edges[:, 1], "sum")
    assert rel_err(base_sum.cpu().numpy(), want) <= RTOL


def test_dynamic_task_queue_large_graph(pgl):
    """More tasks than resident warps (the persistent grid is 2 CTAs per SM): 3M edges at T = 32 * k, repeat launches
    bit-identical."""
    n, e, d = 200000, 3000000, 128
    edges = O.chung_lu_edges(n, e, exponent=0.8, seed=351)
    g = make_graph(pgl, edges, n)
    x = torch.randn(n, d, device="cuda")
    with torch.no_grad():
        base = g._send_u_recv(x, "sum", None)
        for _ in range(2):
            assert torch.equal(g._send_u_recv(x, "sum", None), base)
        a = torch.randn(n, 8, device="cuda")
        gb = pgl.ops.gat_fused(g._fwd_csr(), x.reshape(n, 8, 16), a, a, 0.2)
        for _ in range(2):
            assert torch.equal(pgl.ops.gat_fused(g._fwd_csr(), x.reshape(n, 8, 16), a, a, 0.2), gb)


# ---------------------------------------------------------------- attention projections
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 8), (1, 128), (32, 4), (12, 8), (2, 64)])
def test_head_dots_match_the_two_torch_expressions(pgl, H, Dh):
    """pglb_head_dots_f32 == (sum(f * w_src, -1), sum(f * w_dst, -1)) of pgl/nn/conv.py:323-326, forward and backward."""
    n = 5003
    gen = torch.Generator(device="cuda").manual_seed(360 + H)
    f1 = torch.randn(n, H, Dh, device="cuda", generator=gen).requires_grad_(True)
    ws1 = torch.randn(H, Dh, device="cuda", generator=gen).requires_grad_(True)
    wd1 = torch.randn(H, Dh, device="cuda", generator=gen).requires_grad_(True)
    gs = torch.randn(n, H, device="cuda", generator=gen)
    gd = torch.randn(n, H, device="cuda", generator=gen)
    got = pgl.ops.head_dots(f1, ws1, wd1)
    assert got is not None
    (got[0] * gs + got[1] * gd).sum().backward()
    f2, ws2, wd2 = [t.detach().clone().requires_grad_(True) for t in (f1, ws1, wd1)]
    want = (torch.sum(f2 * ws2, dim=-1), torch.sum(f2 * wd2, dim=-1))
    (want[0] * gs + want[1] * gd).sum().backward()
    for a, b in zip(got, want):
        assert rel_err(a.detach().cpu().numpy(), b.detach().cpu().numpy()) <= 1e-6
    for a, b in ((f1, f2), (ws1, ws2), (wd1, wd2)):
        assert rel_err(a.grad.cpu().numpy(), b.grad.cpu().numpy()) <= 1e-5
    # shapes outside the kernel: the caller keeps the torch expressions
    assert pgl.ops.head_dots(torch.randn(10, 8, 12, device="cuda"), torch.randn(8, 12, device="cuda"),
                             torch.randn(8, 12, device="cuda")) is None          # head_dim not a power of two
    assert pgl.ops.head_dots(torch.randn(10, 16, 16, device="cuda"), torch.randn(16, 16, device="cuda"),
                             torch.randn(16, 16, device="cuda")) is None         # 256 floats per row
    assert pgl.ops.head_dots(f1.double(), ws1, wd1) is None
