"""GATConv's fused training path with attention dropout (the *_drop_* GAT entries).

Contract: with keep bits m (the Philox stream of include/pglb.h, keyed by dst-CSR slot and head) and s = 1 / (1 - p),
out[d] = sum_j s m_j alpha_j f[src_j].  The online softmax's running sum keeps every slot, so lse is bitwise the lse
without dropout; the edge backward returns beta = m ? fl(alpha s) : 0 in place of alpha.  The references below are
plain torch fp32 with the same mask, which comes from the library's host entry (pinned to a numpy restatement of
Philox by tests/test_gat_dropout_host.py) mapped from slot order to edge order through the CSR's edge ids."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
RTOL = 1e-4
DTYPES = (torch.bfloat16, torch.float16)
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
EMPTY = 64   # trailing nodes without an edge: empty rows
SEED = (0x5EED0123456789AB, 4 * 1000)


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


@pytest.fixture(scope="module")
def graph(pgl):
    """Rows cut across tasks (in-degree > 2048), one-edge rows and empty rows (as tests/test_gpu_gat_half.py)."""
    n = 3000
    edges = O.chung_lu_edges(n, 80000, exponent=0.9, seed=301)
    g = pgl.Graph(edges=edges, num_nodes=n + EMPTY)
    g.tensor()
    deg = np.bincount(edges[:, 1], minlength=n + EMPTY)
    assert deg.max() > 2048 and (deg == 0).sum() >= EMPTY and (deg == 1).sum() > 0
    return g, edges


def _bits(t):
    return t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def _rand(shape, seed, dtype=torch.float32):
    return torch.randn(shape, device="cuda", generator=torch.Generator("cuda").manual_seed(seed)).to(dtype)


def rel_err(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max() / max(float(b.abs().max()), 1e-12))


def _s32(p):
    return float(np.float32(1.0 / (1.0 - float(np.float32(p)))))


def edge_mask(pgl, csr, H, p, seed=SEED):
    """[E, H] float32 keep mask in edge order."""
    from pgl_b200 import _lib
    E = int(csr["cols"].shape[0])
    w = np.zeros(E, np.uint32)
    _lib.check(_lib.lib.pglb_attn_dropout_keep_host(seed[0], seed[1], p, 0, E, H, w.ctypes.data_as(ctypes.c_void_p)))
    bits = ((w[:, None] >> np.arange(H, dtype=np.uint32)) & 1).astype(np.float32)
    eid = csr.get("eid")
    m = np.empty_like(bits)
    m[np.arange(E) if eid is None else eid.cpu().numpy()] = bits
    return torch.from_numpy(m).cuda()


def torch_gat_drop(f, a_s, a_d, src, dst, n, slope, mask=None, s=1.0):
    """sum_j s m_j softmax_j(leaky(a_s[src_j,h] + a_d[d,h])) f[src_j,h,:] in plain torch (differentiable)."""
    z = torch.nn.functional.leaky_relu(a_s[src] + a_d[dst], slope)
    H = z.shape[1]
    m = torch.full((n, H), -float("inf"), device=z.device).scatter_reduce(0, dst[:, None].expand(-1, H), z, "amax")
    pe = torch.exp(z - m[dst])
    al = pe / torch.zeros((n, H), device=z.device).index_add(0, dst, pe)[dst]
    beta = al if mask is None else al * mask * torch.tensor(s, dtype=torch.float32, device=z.device)
    return torch.zeros_like(f).index_add(0, dst, f[src] * beta.unsqueeze(-1)), al


def fwd_raw(pgl, csr, f2, a_s, a_d, slope, H, Dh, drop=None):
    """The train entry of f2's dtype, with dropout when drop = (p, seed, offset): (out, lse)."""
    ops = pgl.ops
    lib = ops.lib
    n_src, E, n_dst = int(f2.shape[0]), int(csr["cols"].shape[0]), int(csr["indptr"].shape[0]) - 1
    out = torch.empty((n_dst, H * Dh), dtype=f2.dtype, device="cuda")
    lse = torch.zeros((n_dst, H), dtype=torch.float32, device="cuda")
    ws = ops.workspace(f2.device, 1 << 28)
    args = (ops._ptr(csr["indptr"]), ops._ptr(csr["cols"]), ops._ptr(f2), f2.stride(0), ops._ptr(a_s), ops._ptr(a_d),
            float(slope), ops._ptr(out), out.stride(0), ops._ptr(lse), n_dst, n_src, E, H, Dh)
    tail = (ops._ptr(ws), ws.numel(), ops._stream())
    dt = () if f2.dtype == torch.float32 else (ops._DTYPE16[f2.dtype],)
    if drop is None:
        entry = lib.pglb_gat_fused_train_csr_f32 if not dt else lib.pglb_gat_fused_train_csr_x16
        ops.check(entry(*args, *dt, *tail))
    else:
        entry = lib.pglb_gat_fused_train_drop_csr_f32 if not dt else lib.pglb_gat_fused_train_drop_csr_x16
        ops.check(entry(*args, *dt, *drop, *tail))
    return out, lse


def bwd_raw(pgl, fwd, f, go, out, a_s, a_d, lse, slope, H, Dh, drop=None):
    """The edge backward entry of f's dtype: (alpha_e, dz_e) in edge order."""
    ops = pgl.ops
    E = int(fwd["cols"].shape[0])
    alpha = torch.empty((E, H), device="cuda")
    dz = torch.empty((E, H), device="cuda")
    args = (ops._ptr(fwd["rows"]), ops._ptr(fwd["cols"]), ops._ptr(fwd["eid"]), ops._ptr(f), f.stride(0), ops._ptr(go),
            go.stride(0), ops._ptr(out), out.stride(0), ops._ptr(a_s), ops._ptr(a_d), ops._ptr(lse), slope, E, H, Dh)
    tail = (ops._ptr(alpha), ops._ptr(dz), ops._stream())
    dt = () if f.dtype == torch.float32 else (ops._DTYPE16[f.dtype],)
    if drop is None:
        entry = ops.lib.pglb_gat_bwd_edge_f32 if not dt else ops.lib.pglb_gat_bwd_edge_x16
        ops.check(entry(*args, *dt, *tail))
    else:
        entry = ops.lib.pglb_gat_bwd_edge_drop_f32 if not dt else ops.lib.pglb_gat_bwd_edge_drop_x16
        ops.check(entry(*args, *dt, *drop, *tail))
    return alpha, dz


# 1. forward against torch with the same mask; lse untouched by dropout ------------------------------------------------
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 32), (16, 8), (12, 8)])
@pytest.mark.parametrize("p", [0.1, 0.6])
@pytest.mark.parametrize("warm", ["0", "1"])   # launches before the checked one: each launch re-arms the task queue head
def test_forward_matches_torch_with_the_same_mask(pgl, graph, H, Dh, p, warm):
    g, edges = graph
    csr = g._fwd_csr()
    N = int(g.num_nodes)
    f = _rand((N, H * Dh), 501 + H)
    a_s, a_d = _rand((N, H), 502), _rand((N, H), 503)
    first = [fwd_raw(pgl, csr, f, a_s, a_d, 0.2, H, Dh, drop=(p,) + SEED)[0] for _ in range(int(warm))]
    out, lse = fwd_raw(pgl, csr, f, a_s, a_d, 0.2, H, Dh, drop=(p,) + SEED)
    assert all(torch.equal(o, out) for o in first)
    _, lse0 = fwd_raw(pgl, csr, f, a_s, a_d, 0.2, H, Dh)
    assert torch.equal(lse.view(torch.int32), lse0.view(torch.int32))
    src, dst = torch.from_numpy(edges[:, 0]).cuda(), torch.from_numpy(edges[:, 1]).cuda()
    mask = edge_mask(pgl, csr, H, p)
    ref, _ = torch_gat_drop(f.reshape(N, H, Dh), a_s, a_d, src, dst, N, 0.2, mask, _s32(p))
    assert rel_err(out, ref.reshape(N, -1)) <= RTOL
    assert abs(float(mask.mean()) - (1 - p)) < 0.01


# 2. bit anchors -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H,Dh", [(8, 16), (16, 8)])
def test_bit_anchors(pgl, graph, H, Dh):
    g, _ = graph
    fwd = g._fwd_csr()
    N = int(g.num_nodes)
    f = _rand((N, H * Dh), 511)
    go = _rand((N, H * Dh), 512)
    a_s, a_d = _rand((N, H), 513), _rand((N, H), 514)
    # p = 1e-12: thresh 0 and s = 1.0f, every slot kept: bitwise the entries without dropout
    tiny = (1e-12,) + SEED
    out0, lse0 = fwd_raw(pgl, fwd, f, a_s, a_d, 0.2, H, Dh)
    out1, lse1 = fwd_raw(pgl, fwd, f, a_s, a_d, 0.2, H, Dh, drop=tiny)
    assert torch.equal(_bits(out1), _bits(out0)) and torch.equal(_bits(lse1), _bits(lse0))
    al0, dz0 = bwd_raw(pgl, fwd, f, go, out0, a_s, a_d, lse0, 0.2, H, Dh)
    al1, dz1 = bwd_raw(pgl, fwd, f, go, out1, a_s, a_d, lse1, 0.2, H, Dh, drop=tiny)
    assert torch.equal(_bits(al1), _bits(al0)) and torch.equal(_bits(dz1), _bits(dz0))
    # the same (seed, offset) twice: equal; another offset: another mask
    drop = (0.6,) + SEED
    out2, _ = fwd_raw(pgl, fwd, f, a_s, a_d, 0.2, H, Dh, drop=drop)
    out3, _ = fwd_raw(pgl, fwd, f, a_s, a_d, 0.2, H, Dh, drop=drop)
    out4, _ = fwd_raw(pgl, fwd, f, a_s, a_d, 0.2, H, Dh, drop=(0.6, SEED[0], SEED[1] + 4))
    assert torch.equal(_bits(out2), _bits(out3)) and not torch.equal(out2, out4)
    # the drop backward's alpha_e: exactly 0 where the mask drops, fl(alpha * s) where it keeps
    al2, dz2 = bwd_raw(pgl, fwd, f, go, out2, a_s, a_d, lse0, 0.2, H, Dh, drop=drop)
    al3, dz3 = bwd_raw(pgl, fwd, f, go, out2, a_s, a_d, lse0, 0.2, H, Dh, drop=drop)
    assert torch.equal(_bits(al2), _bits(al3)) and torch.equal(_bits(dz2), _bits(dz3))
    mask = edge_mask(pgl, fwd, H, 0.6) > 0
    s = torch.tensor(_s32(0.6), dtype=torch.float32, device="cuda")
    assert torch.equal(_bits(al2[mask]), _bits(al0[mask] * s))
    assert bool((al2[~mask] == 0).all()) and bool((~mask).any())


# 3. gradients against torch autograd on the same mask ------------------------------------------------------------------
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 32), (16, 8), (12, 8)])
@pytest.mark.parametrize("slope", [0.2, 1.0])
def test_gradients_against_torch(pgl, graph, H, Dh, slope):
    """The bars of test_gat_fused_train_forward_and_gradients."""
    g, edges = graph
    N = int(g.num_nodes)
    p = 0.6
    src, dst = torch.from_numpy(edges[:, 0]).cuda(), torch.from_numpy(edges[:, 1]).cuda()
    f1 = _rand((N, H, Dh), 521).requires_grad_(True)
    s1 = _rand((N, H), 522).requires_grad_(True)
    d1 = _rand((N, H), 523).requires_grad_(True)
    go = _rand((N, H, Dh), 524)
    out = pgl.ops.gat_fused_train(g._fwd_csr(), g._bwd_csr, f1, s1, d1, slope, attn_drop=p, seed=SEED)
    assert out is not None
    out.backward(go)
    f2, s2, d2 = [t.detach().clone().requires_grad_(True) for t in (f1, s1, d1)]
    ref, _ = torch_gat_drop(f2, s2, d2, src, dst, N, slope, edge_mask(pgl, g._fwd_csr(), H, p), _s32(p))
    ref.backward(go)
    assert rel_err(out, ref) <= RTOL, "forward"
    assert rel_err(f1.grad, f2.grad) <= RTOL, "grad f"
    scale = float(s2.grad.abs().max())
    assert float((s1.grad - s2.grad).abs().max()) <= 5e-4 * scale, "grad attn_src"
    assert float((d1.grad - d2.grad).abs().max()) <= 5e-4 * max(scale, float(d2.grad.abs().max())), "grad attn_dst"


# 4. 16-bit: the fp32 drop kernels on the widened inputs ---------------------------------------------------------------
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("H,Dh", [(8, 16), (4, 32), (16, 8), (12, 8)])
def test_x16_is_the_fp32_drop_kernel_on_widened_inputs(pgl, graph, dtype, H, Dh):
    g, _ = graph
    fwd = g._fwd_csr()
    N = int(g.num_nodes)
    f = _rand((N, H * Dh), 531 + H, dtype)
    go = _rand((N, H * Dh), 532, dtype)
    a_s, a_d = _rand((N, H), 533), _rand((N, H), 534)
    drop = (0.6,) + SEED
    out16, lse16 = fwd_raw(pgl, fwd, f, a_s, a_d, 0.2, H, Dh, drop=drop)
    out32, lse32 = fwd_raw(pgl, fwd, f.float(), a_s, a_d, 0.2, H, Dh, drop=drop)
    assert torch.equal(_bits(out16), _bits(out32.to(dtype))) and torch.equal(_bits(lse16), _bits(lse32))
    al16, dz16 = bwd_raw(pgl, fwd, f, go, out16, a_s, a_d, lse16, 0.2, H, Dh, drop=drop)
    al32, dz32 = bwd_raw(pgl, fwd, f.float(), go.float(), out16.float(), a_s, a_d, lse16, 0.2, H, Dh, drop=drop)
    assert torch.equal(_bits(al16), _bits(al32)) and torch.equal(_bits(dz16), _bits(dz32))


# 5. the layer ----------------------------------------------------------------------------------------------------------
DROP_ENTRIES = ("pglb_gat_fused_train_drop_csr_f32", "pglb_gat_fused_train_drop_csr_x16", "pglb_gat_bwd_edge_drop_f32",
                "pglb_gat_bwd_edge_drop_x16")


def _spy(monkeypatch, ops):
    calls = {k: 0 for k in DROP_ENTRIES}
    for name in DROP_ENTRIES:
        real = getattr(ops.lib, name)

        def spy(*a, _real=real, _name=name):
            calls[_name] += 1
            return _real(*a)
        monkeypatch.setattr(ops.lib, name, spy)
    return calls


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_gatconv_trains_with_attention_dropout_on_the_fused_path(pgl, graph, monkeypatch, dtype):
    g, edges = graph
    ops = pgl.ops
    N = int(g.num_nodes)
    torch.manual_seed(3)
    layer = pgl.nn.GATConv(24, 16, feat_drop=0.0, attn_drop=0.6, num_heads=8).cuda().to(dtype).train()
    x = torch.randn(N, 24, device="cuda").to(dtype)
    go = torch.randn(N, 128, device="cuda").to(dtype)
    g._fwd_csr(), g._bwd_csr()   # the one-off index builds are not part of a layer's launch count
    sfx = "f32" if dtype == torch.float32 else "x16"

    def run(seed, fused=True):
        old = ops.GAT_FUSED_TRAIN
        ops.GAT_FUSED_TRAIN = fused
        try:
            torch.manual_seed(seed)
            layer.zero_grad()
            xi = x.clone().requires_grad_(True)
            l0 = ops.launch_count()
            out = layer(g, xi)
            n_launch = ops.launch_count() - l0
            out.backward(go)
            return out.detach(), xi.grad, [p.grad.clone() for p in layer.parameters()], n_launch
        finally:
            ops.GAT_FUSED_TRAIN = old

    calls = _spy(monkeypatch, ops)
    out_a, gx_a, gp_a, n_f = run(11)
    assert calls["pglb_gat_fused_train_drop_csr_" + sfx] == 1 and calls["pglb_gat_bwd_edge_drop_" + sfx] == 1
    # under one torch.manual_seed: bitwise the same outputs and gradients
    out_b, gx_b, gp_b, _ = run(11)
    assert torch.equal(out_a, out_b) and torch.equal(gx_a, gx_b)
    assert all(torch.equal(a, b) for a, b in zip(gp_a, gp_b))
    out_c, _, _, _ = run(12)
    assert not torch.equal(out_a, out_c)
    _, _, _, n_u = run(11, fused=False)
    assert n_f < n_u
    assert out_a.dtype == dtype and gx_a.dtype == dtype

    # unbiased: the mean over K masks tends to the attn_drop = 0 output.  Per element the dropped output is
    # sum_e s m_e alpha_e f_e with Var = p / (1 - p) sum_e alpha_e^2 f_e^2; the mean of K independent masks lies within
    # 6 sqrt(Var / K) of the undropped output, plus the arithmetic error of each sample (2 u |sample| for 16-bit
    # outputs, 1e-5 |sample| for fp32: the kernel's exp is __expf).  And the deviations, in units of that sigma, have
    # the median of a normal's |Z| (0.67), not more: a bias well inside the 6 sigma bar would still show there.
    K, p = 64, 0.6
    with torch.no_grad():
        acc = torch.zeros(N, 128, device="cuda", dtype=torch.float64)
        big = 0.0
        for k in range(K):
            torch.manual_seed(1000 + k)
            o = layer(g, x)
            acc += o.double()
            big = max(big, float(o.abs().max()))
        mean = acc / K
        layer.attn_drop = 0.0
        out0 = layer(g, x).double()
        layer.attn_drop = p
        f = (x.double() @ layer.linear.weight.double() + layer.linear.bias.double()).reshape(N, 8, 16)
        src_e, dst_e = torch.from_numpy(edges[:, 0]).cuda(), torch.from_numpy(edges[:, 1]).cuda()
        z = torch.nn.functional.leaky_relu((f * layer.weight_src.double()).sum(-1)[src_e] +
                                           (f * layer.weight_dst.double()).sum(-1)[dst_e], 0.2)
        pe = torch.exp(z - torch.full((N, 8), -math.inf, device="cuda", dtype=torch.float64).scatter_reduce(
            0, dst_e[:, None].expand(-1, 8), z, "amax")[dst_e])
        al = pe / torch.zeros((N, 8), device="cuda", dtype=torch.float64).index_add(0, dst_e, pe)[dst_e]
        var = torch.zeros((N, 8, 16), device="cuda", dtype=torch.float64).index_add(
            0, dst_e, (al[:, :, None] * f[src_e]) ** 2) * (p / (1 - p))
        sigma = torch.sqrt(var.reshape(N, 128) / K)
        tol = (1e-5 if dtype == torch.float32 else 2 * U[dtype]) * big
        dev = (mean - out0).abs()
        assert bool((dev <= 6 * sigma + tol).all()), float((dev / (6 * sigma + tol)).max())
        z = (dev / sigma)[sigma > 0]
        assert float(z.median()) < 1.0, float(z.median())

    # .eval() ignores attention dropout
    layer.eval()
    with torch.no_grad():
        assert torch.equal(layer(g, x).double(), out0)


@pytest.mark.parametrize("path", ["fused_fp32", "op_by_op_fp32", "fused_bf16"])
def test_training_with_attention_dropout_learns(pgl, graph, path):
    """The task of test_bf16_training_tracks_fp32 (GATConv(32 -> 8 x 16) + a linear classifier, 40 Adam steps) with
    attn_drop = 0.6: the eval-mode loss falls below 0.7 x its value at the start."""
    g, _ = graph
    ops = pgl.ops
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
            self.c1 = nn.GATConv(32, 16, feat_drop=0.0, attn_drop=0.6, num_heads=8)
            self.out = torch.nn.Linear(128, 6)

        def forward(self, h):
            return self.out(self.c1(g, h))

    torch.manual_seed(2)
    net = Net().cuda()
    xin = x
    if path == "fused_bf16":
        net, xin = net.to(torch.bfloat16), x.to(torch.bfloat16)

    def eval_loss():
        net.eval()
        with torch.no_grad():
            v = float(torch.nn.functional.cross_entropy(net(xin).float(), y))
        net.train()
        return v

    old = ops.GAT_FUSED_TRAIN
    ops.GAT_FUSED_TRAIN = path != "op_by_op_fp32"
    try:
        l0 = eval_loss()
        opt = torch.optim.Adam(net.parameters(), lr=1e-2)
        for _ in range(40):
            opt.zero_grad()
            torch.nn.functional.cross_entropy(net(xin).float(), y).backward()
            opt.step()
        l1 = eval_loss()
    finally:
        ops.GAT_FUSED_TRAIN = old
    assert l1 < 0.7 * l0, (l0, l1)


def test_declines(pgl, graph):
    """attn_drop >= 1, shapes outside the kernels and graph capture return None (the caller stays op-by-op)."""
    g, _ = graph
    N = int(g.num_nodes)
    f = _rand((N, 8, 16), 541).requires_grad_(True)
    a = _rand((N, 8), 542)
    assert pgl.ops.gat_fused_train(g._fwd_csr(), g._bwd_csr, f, a, a, 0.2, attn_drop=1.0) is None
    f4 = _rand((N, 4, 8), 543).requires_grad_(True)
    assert pgl.ops.gat_fused_train(g._fwd_csr(), g._bwd_csr, f4, a[:, :4], a[:, :4], 0.2, attn_drop=0.5) is None
    # the default stream draws from the CUDA default generator and advances its offset by 4 per call
    gen = torch.cuda.default_generators[torch.cuda.current_device()]
    torch.manual_seed(9)
    off0 = gen.get_offset()
    pgl.ops.gat_fused_train(g._fwd_csr(), g._bwd_csr, f, a, a, 0.2, attn_drop=0.5)
    assert gen.get_offset() == off0 + 4
    # an op-by-op fallback layer (H % 4) still trains with its nn.Dropout
    layer = pgl.nn.GATConv(16, 8, feat_drop=0.0, attn_drop=0.5, num_heads=2).cuda().train()
    xx = torch.randn(N, 16, device="cuda", requires_grad=True)
    layer(g, xx).sum().backward()
    assert torch.isfinite(xx.grad).all()
