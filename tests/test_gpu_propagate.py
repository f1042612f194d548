"""The fused K-hop propagation step (pglb_propagate_f32 / pglb_propagate_narrow_f32, ops.propagate) and the layers
that run on it (APPNP, GCNII, SSGCConv, GPRConv).

Contract (include/pglb.h): with t the row send_u_recv(sum, scale_src = scale_dst = norm) writes on the same route,
y = a t (+ b h), acc_out = acc_in + c y, every product and sum rounded on its own.  On dyadic inputs every value is
exact in float32, so the kernels must equal a float64 numpy restatement bit for bit; on random data the fused hop must
equal the op-by-op torch hop bit for bit."""
import numpy as np
import pytest
import torch

from oracle import oracle as O

pytestmark = pytest.mark.gpu
DIMS = [1, 7, 16, 40, 47, 64, 100, 128, 129, 256, 1433]
N = 3000
EMPTY = 50      # trailing nodes without an in-edge
HUB_DEG = 1500  # in-edges of node 0: the node-parallel hub path and a row cut across wide-row / narrow tasks
GRAD_TOL = 1e-4


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


def _edges(seed=7):
    e = O.chung_lu_edges(N, 40000, exponent=0.8, seed=seed)
    e = e[e[:, 1] < N - EMPTY]
    rng = np.random.default_rng(seed)
    hub = np.stack([rng.integers(0, N, HUB_DEG), np.zeros(HUB_DEG, np.int64)], 1)
    one = np.stack([rng.integers(0, N, 20), np.arange(N - EMPTY - 20, N - EMPTY)], 1)   # rows of one edge
    keep = ~np.isin(e[:, 1], np.arange(N - EMPTY - 20, N - EMPTY))
    return np.concatenate([e[keep], hub, one]).astype(np.int64)


@pytest.fixture(scope="module")
def graph(pgl):
    e = _edges()
    g = pgl.Graph(edges=e, num_nodes=N)
    g.tensor()
    deg = np.bincount(e[:, 1], minlength=N)
    assert deg[0] > 1024 and (deg == 0).sum() >= EMPTY and (deg == 1).sum() >= 20
    return g, e


def _fwd(g):
    return g._fwd_csr()


def _ref(e, x, ns, a, b=None, h=None, acc=None, c=None):
    """float64 restatement of the contract"""
    x = x.astype(np.float64)
    t = np.zeros_like(x)
    np.add.at(t, e[:, 1], ns[e[:, 0], None] * x[e[:, 0]])
    t = t * ns[:, None]
    y = a * t + (b * h if h is not None else 0.0)
    return y, (acc + c * y if acc is not None else None)


def _dyadic(rng, shape):
    return rng.integers(-2, 3, shape).astype(np.float32)


@pytest.mark.parametrize("D", DIMS)
def test_exact_contract(pgl, graph, D):
    g, e = graph
    rng = np.random.default_rng(D)
    x = _dyadic(rng, (N, D))
    hv = _dyadic(rng, (N, D))
    av = _dyadic(rng, (N, D))
    ns = (2.0 ** rng.integers(-2, 1, N)).astype(np.float32)
    xd, hd, nd = (torch.from_numpy(v).cuda() for v in (x, hv, ns))
    for a, b, c in [(0.75, 0.25, -1.0), (-2.0, -1.0, 0.5), (0.5, -0.25, 0.75)]:
        for h_kind in ("none", "h", "x"):
            h = {"none": None, "h": hd, "x": xd}[h_kind]
            hn = {"none": None, "h": hv, "x": x}[h_kind]
            for acc_kind in ("none", "out", "inplace", "c_dev"):
                acc = None if acc_kind == "none" else torch.from_numpy(av).cuda()
                cc = torch.tensor([c], device="cuda") if acc_kind == "c_dev" else c
                with torch.no_grad():
                    r = pgl.ops.propagate(xd, _fwd(g), None, nd, a=a, b=b, h=h, acc=acc, c=cc,
                                          inplace_acc=acc_kind == "inplace")
                if D == 256:
                    # 16-byte rows past 128 elements take spmm_stream, which has no epilogue: the call declines
                    assert r is None
                    continue
                assert r is not None
                y, ao = (r, None) if acc is None else r
                if acc_kind == "inplace":
                    assert ao is acc
                wy, wa = _ref(e, x, ns.astype(np.float64), a, b, hn, av if acc is not None else None, c)
                np.testing.assert_array_equal(y.cpu().numpy().astype(np.float64), wy, err_msg="%s %s" % (h_kind,
                                                                                                      acc_kind))
                if acc is not None:
                    np.testing.assert_array_equal(ao.cpu().numpy().astype(np.float64), wa)


@pytest.mark.parametrize("D", [7, 40, 47, 129])
def test_strided_unaligned_x(pgl, graph, D):
    g, e = graph
    rng = np.random.default_rng(100 + D)
    big = torch.from_numpy(_dyadic(rng, (N, D + 3))).cuda()
    xs = big[:, 1:D + 1]            # row stride D + 3, 4-byte offset: the node-parallel kernel, one element per lane
    ns = (2.0 ** rng.integers(-2, 1, N)).astype(np.float32)
    nd = torch.from_numpy(ns).cuda()
    y = pgl.ops._propagate_raw(_fwd(g), xs, nd, 0.5, 0.0, None, None, 1.0, None)
    wy, _ = _ref(e, xs.cpu().numpy(), ns.astype(np.float64), 0.5)
    np.testing.assert_array_equal(y.cpu().numpy().astype(np.float64), wy)


def _op_hop_appnp(graph, feature, norm, h0, alpha):
    from pgl_b200.nn.conv import _propagate
    feature = _propagate(graph, feature, norm)
    return alpha * h0 + (1 - alpha) * feature


def _appnp_ref(pgl, g, x, alpha, k, norm=None, self_loop=False):
    from pgl_b200.nn.conv import _with_self_loops
    import pgl_b200.nn.functional as GF
    if self_loop:
        g = _with_self_loops(g)
    if norm is None:
        norm = GF.degree_norm(g)
    f = x
    for _ in range(k):
        f = _op_hop_appnp(g, f, norm, x, alpha)
    return f


def _eq(a, b):
    assert torch.equal(a, b), (a - b).abs().max().item()


@pytest.mark.parametrize("D", DIMS)
def test_layers_bit_identical_to_op_by_op(pgl, graph, D):
    from pgl_b200.nn import conv as C
    import pgl_b200.nn.functional as GF
    g, _ = graph
    torch.manual_seed(D)
    x = torch.randn(N, D, device="cuda")
    norm_c = torch.rand(N, 1, device="cuda") + 0.5
    for grad in (False, True):
        xg = x.clone().requires_grad_(grad)
        with torch.set_grad_enabled(grad):
            _eq(C.APPNP(alpha=0.1, k_hop=10)(g, xg), _appnp_ref(pgl, g, xg, 0.1, 10))
            _eq(C.APPNP(alpha=0.1, k_hop=10)(g, xg, norm_c), _appnp_ref(pgl, g, xg, 0.1, 10, norm=norm_c))
            _eq(C.APPNP(alpha=0.1, k_hop=10, self_loop=True)(g, xg), _appnp_ref(pgl, g, xg, 0.1, 10, self_loop=True))
            # GCNII (eval: dropout off) against its hops restated
            m = C.GCNII(D, activation="relu", k_hop=8).cuda().eval()
            norm = GF.degree_norm(g)
            f = xg
            for i in range(8):
                beta = np.log(0.5 / (i + 1) + 1)
                f = _op_hop_appnp(g, f, norm, xg, m.alpha)
                f = torch.relu(beta * m.mlps[i](f) + (1 - beta) * f)
            _eq(m(g, xg), f)
            # SSGCConv smoothing
            s = C.SSGCConv(D, 3, k_hop=16, cached=False).cuda()
            f, acc = xg, xg
            for _ in range(16):
                f = (1 - s.alpha) * C._propagate(g, f, norm)
                acc = acc + f
            _eq(s._smooth(g, xg), acc / 16 + s.alpha * xg)
            # GPRConv's hops (PPR, k = 10) from the same MLP output
            gp = C.GPRConv(D, 8, D, drop=0.0, dprate=0.0, k_hop=10).cuda().eval()
            f = gp.linear_2(torch.relu(gp.linear_1(xg)))
            hid = f * gp.temp[0]
            for k in range(10):
                f = C._propagate(g, f, norm)
                hid = hid + gp.temp[k + 1] * f
            _eq(gp(g, xg), hid)


@pytest.mark.parametrize("D", [16, 47, 128])
def test_chebnet_and_bernnet_recurrences(pgl, graph, D):
    from pgl_b200.nn.conv import _propagate
    import pgl_b200.nn.functional as GF
    g, _ = graph
    norm = GF.degree_norm(g)
    torch.manual_seed(3)
    x = torch.randn(N, D, device="cuda")
    with torch.no_grad():
        # ChebNetII: T_k = -2 A T_{k-1} - T_{k-2}
        t0, t1 = x, _propagate(g, x, norm)
        f0, f1 = t0, t1
        for _ in range(4):
            t0, t1 = t1, -2 * _propagate(g, t1, norm) - t0
            f0, f1 = f1, pgl.ops.propagate(f1, _fwd(g), None, norm, a=-2.0, b=-1.0, h=f0)
            _eq(f1, t1)
        # BernNet: (I + A) x, h aliasing x
        _eq(pgl.ops.propagate(x, _fwd(g), None, norm, a=1.0, b=1.0, h=x), x + _propagate(g, x, norm))


def _dense_ref(e, x64, ns64):
    src, dst = torch.from_numpy(e[:, 0]).cuda(), torch.from_numpy(e[:, 1]).cuda()
    t = torch.zeros_like(x64).index_add(0, dst, ns64[src, None] * x64[src])
    return t * ns64[:, None]


@pytest.mark.parametrize("D", [7, 64, 128, 129])
def test_gradients(pgl, graph, D):
    from pgl_b200.nn import conv as C
    import pgl_b200.nn.functional as GF
    g, e = graph
    torch.manual_seed(11)
    norm = GF.degree_norm(g).reshape(-1)
    x = torch.randn(N, D, device="cuda", requires_grad=True)
    h0 = torch.randn(N, D, device="cuda", requires_grad=True)
    temp = torch.rand(4, device="cuda", requires_grad=True)
    w = torch.randn(N, D, device="cuda")

    def fused():
        f, acc = x, h0 * temp[0]
        for k in range(3):
            f = pgl.ops.propagate(f, _fwd(g), g._bwd_csr, norm, a=0.9, b=0.1, h=h0)
            f, acc = pgl.ops.propagate(f, _fwd(g), g._bwd_csr, norm, acc=acc, c=temp[k + 1])
        return ((f + acc) * w).sum()

    def ref():
        x64, h64, t64 = (v.detach().double().requires_grad_(True) for v in (x, h0, temp))
        f, acc = x64, h64 * t64[0]
        for k in range(3):
            f = 0.9 * _dense_ref(e, f, norm.double()) + 0.1 * h64
            f = _dense_ref(e, f, norm.double())
            acc = acc + t64[k + 1] * f
        ((f + acc) * w.double()).sum().backward()
        return x64.grad, h64.grad, t64.grad

    grads = []
    for _ in range(2):
        for v in (x, h0, temp):
            v.grad = None
        fused().backward()
        grads.append([v.grad.clone() for v in (x, h0, temp)])
    for a, b in zip(*grads):
        assert torch.equal(a, b)   # no atomics: the same bits run to run
    for got, want in zip(grads[0], ref()):
        err = (got.double() - want).abs().max() / want.abs().max()
        assert err <= GRAD_TOL, err.item()


def test_appnp_calls_the_entry_once_per_hop(pgl, graph, monkeypatch):
    from pgl_b200.nn import conv as C
    g, _ = graph
    calls = []
    real = pgl.ops.lib.pglb_propagate_f32

    def counting(*args):
        rc = real(*args)
        calls.append(rc)
        return rc
    monkeypatch.setattr(pgl.ops.lib, "pglb_propagate_f32", counting)
    x = torch.randn(N, 128, device="cuda")
    with torch.no_grad():
        C.APPNP(alpha=0.1, k_hop=10)(g, x)
    assert calls == [0] * 10


def _cuda_kernels(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize("D", [47, 64, 128])
def test_fused_forward_launches(pgl, graph, D):
    from pgl_b200.nn import conv as C
    import pgl_b200.nn.functional as GF
    g, _ = graph
    x = torch.randn(N, D, device="cuda")
    norm = GF.degree_norm(g)
    with torch.no_grad():
        C.APPNP(alpha=0.1, k_hop=2)(g, x)   # warm the graph's caches
        fused2 = _cuda_kernels(lambda: C.APPNP(alpha=0.1, k_hop=2)(g, x))
        fused10 = _cuda_kernels(lambda: C.APPNP(alpha=0.1, k_hop=10)(g, x))
        op10 = _cuda_kernels(lambda: _appnp_ref(pgl, g, x, 0.1, 10, norm=norm))
    torch_kernels = lambda names: [n for n in names if "pglb" not in n and "Memset" not in n]   # noqa: E731
    # nothing but the library's kernels inside the hop loop
    assert len(torch_kernels(fused10)) == len(torch_kernels(fused2))
    assert len(fused10) < len(op10)


def test_declines(pgl, graph):
    from pgl_b200.nn import conv as C
    import pgl_b200.nn.functional as GF
    g, _ = graph
    fwd = _fwd(g)
    norm = GF.degree_norm(g)
    x = torch.randn(N, 16, device="cuda")
    assert pgl.ops.propagate(x.bfloat16(), fwd, None, norm) is None
    assert pgl.ops.propagate(x.double(), fwd, None, norm) is None
    assert pgl.ops.propagate(x.cpu(), fwd, None, norm) is None
    assert pgl.ops.propagate(x[:-1], fwd, None, norm) is None
    assert pgl.ops.propagate(x, fwd, None, norm, h=x[:, :8]) is None
    assert pgl.ops.propagate(x, fwd, None, norm, acc=x.half()) is None
    assert pgl.ops.propagate(x, fwd, None, norm[:-1]) is None
    assert pgl.ops.propagate(x, fwd, None, norm.double()) is None
    ng = norm.clone().requires_grad_(True)
    assert pgl.ops.propagate(x, fwd, None, ng) is None
    assert pgl.ops.propagate(x, dict(fwd, indptr=torch.zeros_like(fwd["indptr"]), cols=fwd["cols"][:0]), None,
                             norm) is None
    # a declined layer call runs the op-by-op hop: the same bits
    _eq(C.APPNP(alpha=0.1, k_hop=3)(g, x, ng), _appnp_ref(pgl, g, x, 0.1, 3, norm=ng))
    xb = x.bfloat16()
    _eq(C.APPNP(alpha=0.1, k_hop=3)(g, xb), _appnp_ref(pgl, g, xb, 0.1, 3))


def _cora_models(C, din, ncls):
    class APPNPNet(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.l1, self.l2 = C.Linear(din, 64), C.Linear(64, ncls)
            self.drop = torch.nn.Dropout(0.5)
            self.prop = C.APPNP(alpha=0.1, k_hop=10)

        def forward(self, g, x):
            return self.prop(g, self.l2(self.drop(torch.relu(self.l1(self.drop(x))))))

    class GCNIINet(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.l1, self.l2 = C.Linear(din, 64), C.Linear(64, ncls)
            self.drop = torch.nn.Dropout(0.6)
            self.conv = C.GCNII(64, activation="relu", lambda_l=0.5, alpha=0.1, k_hop=16, dropout=0.6)

        def forward(self, g, x):
            return self.l2(self.drop(self.conv(g, torch.relu(self.l1(self.drop(x))))))
    return {"APPNP": APPNPNet, "GCNII": GCNIINet}


@pytest.mark.parametrize("model", ["APPNP", "GCNII"])
def test_cora_training_on_both_routes(pgl, model, monkeypatch):
    import os
    from pgl_b200.nn import conv as C
    cora = O.load_cora(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cora.npz"))
    g = pgl.Graph(edges=cora["edges"], num_nodes=cora["num_nodes"])
    g.tensor()
    x = torch.from_numpy(cora["x"]).cuda()
    y = torch.from_numpy(cora["y"]).cuda()
    idx = {k: torch.from_numpy(cora[k + "_index"]).cuda() for k in ("train", "val", "test")}
    net = _cora_models(C, 1433, cora["num_classes"])[model]

    def run(seed):
        torch.manual_seed(seed)
        m = net().cuda()
        opt = torch.optim.Adam(m.parameters(), lr=0.01, weight_decay=5e-4)
        best_val, test_at_best = -1.0, 0.0
        for _ in range(100):
            m.train()
            loss = torch.nn.functional.cross_entropy(m(g, x)[idx["train"]], y[idx["train"]])
            opt.zero_grad()
            loss.backward()
            opt.step()
            m.eval()
            with torch.no_grad():
                pred = m(g, x).argmax(1)
            val = float((pred[idx["val"]] == y[idx["val"]]).float().mean())
            if val > best_val:
                best_val, test_at_best = val, float((pred[idx["test"]] == y[idx["test"]]).float().mean())
        return test_at_best

    fused = np.mean([run(s) for s in range(3)])
    with monkeypatch.context() as mp:
        mp.setattr(pgl.ops, "propagate", lambda *a, **k: None)
        op = np.mean([run(s) for s in range(3)])
    assert fused > 0.5 and abs(fused - op) <= 0.02, (fused, op)
