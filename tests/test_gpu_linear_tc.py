"""pglb_linear_tf32x3_f32 (3xTF32 tensor-core GEMM with fused bias + ReLU, the conv layers' dense
transform, reference pgl/nn/conv.py:238-251) against a float64 matmul.  The bound is 2e-5 relative to
the largest output -- fp32 territory; a single-pass TF32 GEMM sits near 5e-4 and would fail, and the
north_star tolerance for fp32 work is 1e-4."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    return pgl_b200


def rel_err(a, b):
    a = a.double()
    b = b.double()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-12))


@pytest.mark.parametrize("pad", ["8", "16"])   # x read in place from a buffer with `pad` NaN columns after each row
@pytest.mark.parametrize("M,K,N", [(5000, 128, 128), (4097, 100, 128), (10000, 64, 64), (6401, 8, 64),
                                   (64, 128, 128), (1, 4, 128), (70001, 128, 64),
                                   (70001, 128, 128)])
def test_linear_tc_matches_fp64(pgl, M, K, N, pad):
    gen = torch.Generator(device="cuda").manual_seed(M + K + N)
    buf = torch.full((M, K + int(pad)), float("nan"), device="cuda")
    x = buf[:, :K]
    x.copy_(torch.randn(M, K, device="cuda", generator=gen) * 3)
    w = torch.randn(K, N, device="cuda", generator=gen)
    b = torch.randn(N, device="cuda", generator=gen)
    ref = x.double() @ w.double()
    out = pgl.ops._linear_tc_raw(x, w, None, None)
    assert out.shape == (M, N) and rel_err(out, ref) <= 2e-5
    out = pgl.ops._linear_tc_raw(x, w, b, "relu")
    assert rel_err(out, torch.relu(ref + b.double())) <= 2e-5
    assert float(out.min()) >= 0.0
    # and it is at least as close to fp64 as ten times the plain fp32 matmul error
    e_torch = rel_err(x @ w, ref)
    assert rel_err(pgl.ops._linear_tc_raw(x, w, None, None), ref) <= max(10 * e_torch, 2e-6)


def test_linear_tc_strided_input_and_special_values(pgl):
    gen = torch.Generator(device="cuda").manual_seed(7)
    big = torch.randn(9000, 256, device="cuda", generator=gen)
    x = big[:, 64:192]  # row stride 256, 16-byte aligned column offset: read in place
    w = torch.randn(128, 128, device="cuda", generator=gen)
    out = pgl.ops.linear_tc(x, w)
    assert rel_err(out, x.double() @ w.double()) <= 2e-5
    x2 = big[:, 1:129]  # misaligned view: the wrapper makes it contiguous
    assert rel_err(pgl.ops.linear_tc(x2, w), x2.double() @ w.double()) <= 2e-5
    # zeros stay zeros; the identity reproduces x to the 3xTF32 split's 2^-22, not bit for bit
    eye = torch.eye(128, device="cuda")
    xi = torch.randn(4500, 128, device="cuda", generator=gen)
    assert rel_err(pgl.ops.linear_tc(xi, eye), xi) <= 1e-6
    assert torch.equal(pgl.ops.linear_tc(torch.zeros_like(xi), w), torch.zeros(4500, 128, device="cuda"))


def test_linear_tc_errors(pgl):
    from pgl_b200._lib import PglbError
    x = torch.randn(100, 128, device="cuda")
    with pytest.raises(PglbError):
        pgl.ops._linear_tc_raw(x, torch.randn(128, 96, device="cuda"), None, None)
    with pytest.raises(PglbError):
        pgl.ops._linear_tc_raw(torch.randn(100, 130, device="cuda"), torch.randn(130, 128, device="cuda"),
                               None, None)
    assert not pgl.ops.linear_tc_ok(x, torch.randn(128, 128, device="cuda"))  # below the row threshold
    assert pgl.ops.linear_tc_ok(torch.randn(5000, 128, device="cuda"), torch.randn(128, 128, device="cuda"))
    assert not pgl.ops.linear_tc_ok(torch.randn(5000, 128, device="cuda"), torch.randn(128, 16, device="cuda"))


def test_linear_tc_autograd_and_gcn_layer(pgl):
    from oracle import oracle as O
    gen = torch.Generator(device="cuda").manual_seed(11)
    M, K, N = 6000, 64, 128
    x1 = torch.randn(M, K, device="cuda", generator=gen).requires_grad_(True)
    w1 = torch.randn(K, N, device="cuda", generator=gen).requires_grad_(True)
    b1 = torch.randn(N, device="cuda", generator=gen).requires_grad_(True)
    x2, w2, b2 = (t.detach().clone().requires_grad_(True) for t in (x1, w1, b1))
    go = torch.randn(M, N, device="cuda", generator=gen)
    out = pgl.ops.linear_tc(x1, w1, b1, "relu")
    out.backward(go)
    # same ReLU mask on both sides (a pre-activation within rounding of 0 may flip between the two GEMMs)
    ((x2 @ w2 + b2) * (out.detach() > 0)).backward(go)
    for a, b in ((x1, x2), (w1, w2), (b1, b2)):
        assert rel_err(a.grad, b.grad) <= 1e-4
    for t in (x1, w1, b1, x2, w2, b2):
        t.grad = None
    pgl.ops.linear_tc(x1, w1, None, None).backward(go)
    (x2 @ w2).backward(go)
    assert rel_err(x1.grad, x2.grad) <= 1e-4 and rel_err(w1.grad, w2.grad) <= 1e-4 and b1.grad is None
    # GCNConv(128 -> 128, relu) on a graph big enough to take the tensor-core path, vs the oracle
    n, e, d = 6000, 60000, 128
    edges = O.chung_lu_edges(n, e, exponent=0.8, seed=601)
    rng = np.random.default_rng(602)
    x = rng.standard_normal((n, d)).astype(np.float32)
    w = (rng.standard_normal((d, d)) * 0.1).astype(np.float32)
    b = rng.standard_normal(d).astype(np.float32)
    g = pgl.Graph(edges=edges, num_nodes=n)
    g.tensor()
    conv = pgl.nn.GCNConv(d, d, activation="relu").cuda()
    with torch.no_grad():
        conv.linear.weight.copy_(torch.from_numpy(w))
        conv.bias.copy_(torch.from_numpy(b))
        l0 = pgl.ops.launch_count()
        out = conv(g, torch.from_numpy(x).cuda()).cpu().numpy()
    assert pgl.ops.launch_count() > l0
    want = O.gcn_conv(edges, n, x, w, b, activation="relu")
    err = np.abs(out.astype(np.float64) - want).max() / np.abs(want).max()
    assert err <= 1e-4
