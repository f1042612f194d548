"""Graph-level readouts on the device (csrc/readout.cu): segment top-k equal to the numpy oracle on both paths, pad /
unpad bit-exact in four dtypes, the fused attention readout against the float64 oracle from empty segments to 10^6
rows, its determinism, launch count and gradients, the reference's known answers through the public API, and the
pooling layers (the reference's test_pool.py checks, torch restatements of the reference op order, the Set2Set quirk
and a short graph-classification training run)."""
import json
import math
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import oracle_pool as P

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    torch.cuda.set_device(0)
    return pgl_b200


@pytest.fixture(scope="module")
def kat():
    with open(os.path.join(ROOT, "tests", "golden", "kat_readout.json")) as f:
        return json.load(f)


def dev(a, dtype=None):
    return torch.as_tensor(np.asarray(a), dtype=dtype).cuda()


def ids_of(sizes):
    return np.repeat(np.arange(len(sizes)), sizes).astype(np.int64)


def indptr_of(sizes):
    return dev(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64))


def batch_graph(pgl, sizes, seed=0, feat=None):
    rng = np.random.default_rng(seed)
    gs = []
    for n in sizes:
        e = rng.integers(0, n, (2 * n, 2)) if n > 1 else np.zeros((0, 2), np.int64)
        gs.append(pgl.Graph(edges=e, num_nodes=n))
    return pgl.Graph.disjoint(gs).tensor()


# ---- segment top-k ------------------------------------------------------------------------------------------------

def tie_scores(rng, n):
    s = rng.integers(-3, 4, n).astype(np.float32)
    special = np.array([0.0, -0.0, np.nan, -np.inf, np.inf, -1e30, -2e20, 1e-45], np.float32)
    pick = rng.random(n) < 0.2
    s[pick] = rng.choice(special, pick.sum())
    return s


@pytest.mark.parametrize("ratio", [0.3, 0.5, 0.01, 1.0, 1, 3, 100])
def test_topk_equals_oracle_molecule_batch(pgl, ratio):
    rng = np.random.default_rng(7)
    sizes = rng.integers(10, 41, 256)
    sizes[[3, 50, 51]] = 0                     # empty segments inside the batch
    sizes[100] = 1
    ids = ids_of(sizes)
    s = tie_scores(rng, ids.size)
    perm = pgl.ops.segment_topk_perm(dev(s), indptr_of(sizes), ratio)
    assert perm.cpu().numpy().tolist() == P.segment_topk_perm(s, ids, ratio).tolist()


@pytest.mark.parametrize("ratio", [0.3, 0.6, 2])
def test_topk_equals_oracle_long_segment(pgl, ratio):
    rng = np.random.default_rng(8)
    sizes = np.array([30, 0, 100_000, 5, 2049, 0, 17])
    ids = ids_of(sizes)
    s = tie_scores(rng, ids.size)
    perm = pgl.ops.segment_topk_perm(dev(s), indptr_of(sizes), ratio)
    assert perm.cpu().numpy().tolist() == P.segment_topk_perm(s, ids, ratio).tolist()


def test_topk_paths_agree(pgl):
    """The shared-memory path and the radix-sort path give the same perm (the sort path forced by a max_len hint
    above 2048 on a batch whose segments are all short)."""
    import ctypes
    from pgl_b200 import _lib
    rng = np.random.default_rng(9)
    sizes = rng.integers(0, 300, 400)
    ids = ids_of(sizes)
    s = dev(tie_scores(rng, ids.size))
    ip = indptr_of(sizes)
    want = pgl.ops.segment_topk_perm(s, ip, 0.37)
    B, N = len(sizes), int(ids.size)
    offsets = torch.empty(B + 1, dtype=torch.int64, device="cuda")
    info = torch.empty(2, dtype=torch.int64, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.lib.pglb_segment_topk_count(ctypes.c_void_p(ip.data_ptr()), B, 0.37, 0,
                                                ctypes.c_void_p(offsets.data_ptr()), ctypes.c_void_p(info.data_ptr()),
                                                st))
    need = ctypes.c_size_t(0)
    _lib.check(_lib.lib.pglb_segment_topk_ws(B, N, N, ctypes.byref(need)))
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    got = torch.empty(int(info[0].item()), dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib.pglb_segment_topk_fill(ctypes.c_void_p(s.data_ptr()), N, ctypes.c_void_p(ip.data_ptr()), B,
                                               ctypes.c_void_p(offsets.data_ptr()), N,
                                               ctypes.c_void_p(got.data_ptr()), ctypes.c_void_p(ws.data_ptr()),
                                               ws.numel(), st))
    assert torch.equal(got, want)
    assert int(info[1].item()) == int(sizes.max())


def test_segment_topk_public(pgl, kat):
    k = kat["segment_topk"]
    x = dev(np.array(k["data"], np.float32)).requires_grad_(True)
    out, idx = pgl.math.segment_topk(x, dev(np.array(k["scores"], np.float32)), dev(k["segment_ids"]), k["ratio"],
                                     return_index=True)
    assert idx.tolist() == k["index"] and out.tolist() == k["out"]
    out.sum().backward()
    assert x.grad.sum(1).tolist() == [0, 3, 0, 3, 3]
    _, idx = pgl.math.segment_topk(x, dev(np.array(k["scores"], np.float32)), dev(k["segment_ids"]), k["ratio"],
                                   min_score=k["min_score"], return_index=True)
    assert idx.tolist() == k["index_min_score"]
    # the min_score branch against the oracle on a random batch
    rng = np.random.default_rng(4)
    sizes = rng.integers(1, 30, 50)
    ids = ids_of(sizes)
    s = rng.standard_normal(ids.size).astype(np.float32)
    xs = rng.standard_normal((ids.size, 4)).astype(np.float32)
    for ms in (-0.5, 0.3, 5.0):
        out, idx = pgl.math.segment_topk(dev(xs), dev(s), dev(ids), 0.5, min_score=ms, return_index=True)
        wo, wi = P.segment_topk(xs, s, ids, 0.5, min_score=ms)
        assert idx.tolist() == wi.tolist() and np.array_equal(out.cpu().numpy(), wo)


# ---- pad / unpad --------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, torch.float64])
def test_pad_unpad_bit_exact(pgl, dtype):
    rng = np.random.default_rng(11)
    sizes = np.array([3, 0, 7, 1, 0, 12, 5])
    n = int(sizes.sum())
    x = torch.randn(n, 6, 5, dtype=torch.float64, generator=torch.Generator().manual_seed(1)).to(dtype).cuda()
    ip = indptr_of(sizes)
    out = pgl.ops.segment_pad(x, ip, 14, fill_value=-2.5)
    ids = ids_of(sizes)
    pos = np.arange(n) - np.concatenate([[0], np.cumsum(sizes)])[ids]
    want = torch.full((7, 14, 6, 5), -2.5, dtype=dtype, device="cuda")
    want[torch.as_tensor(ids).cuda(), torch.as_tensor(pos).cuda()] = x
    assert out.dtype == dtype and torch.equal(out.view(torch.uint8), want.view(torch.uint8))
    back = pgl.ops.segment_unpad(out, ip, n)
    assert torch.equal(back.view(torch.uint8), x.view(torch.uint8))
    assert rng is not None


def test_pad_unpad_gradients(pgl):
    sizes = np.array([4, 0, 2, 9])
    n = int(sizes.sum())
    ip = indptr_of(sizes)
    x = torch.randn(n, 3, device="cuda", requires_grad=True)
    g = torch.randn(4, 10, 3, device="cuda")
    (pgl.ops.segment_pad(x, ip, 10) * g).sum().backward()
    ids = torch.as_tensor(ids_of(sizes)).cuda()
    pos = torch.arange(n, device="cuda") - ip[ids]
    assert torch.equal(x.grad, g[ids, pos])
    p = torch.randn(4, 10, 3, device="cuda", requires_grad=True)
    gy = torch.randn(n, 3, device="cuda")
    (pgl.ops.segment_unpad(p, ip, n) * gy).sum().backward()
    want = torch.zeros(4, 10, 3, device="cuda")
    want[ids, pos] = gy
    assert torch.equal(p.grad, want)


def test_segment_padding_and_dense_batch_kats(pgl, kat):
    k = kat["segment_padding"]
    out, seq_len, index = pgl.math.segment_padding(dev(np.array(k["data"], np.float32)), dev(k["segment_ids"]))
    assert out.tolist() == k["out"] and seq_len.dtype == torch.int32 and seq_len.tolist() == [2, 0, 1]
    assert index.tolist() == [[0, 0], [0, 1], [2, 0]]
    k = kat["to_dense_batch"]
    from pgl_b200.utils.transform import to_dense_batch
    g = pgl.Graph.disjoint([pgl.Graph(num_nodes=i, edges=[(0, 0)]) for i in k["graph_sizes"]]).tensor()
    x = dev(np.array(k["data"], np.float32))
    out, mask = to_dense_batch(x, g, fill_value=0)
    assert out.tolist() == k["out"] and mask.tolist() == k["mask"] and out.dtype == torch.float32
    out, _ = to_dense_batch(x.double(), g, max_num_nodes=5)
    assert out.dtype == torch.float64 and out.shape == (3, 5, 3)
    with pytest.raises(ValueError):
        to_dense_batch(x, g, max_num_nodes=2)


def test_filter_adj_and_graph_norm_kats(pgl, kat):
    from pgl_b200.utils.transform import filter_adj
    k = kat["filter_adj"]
    e = dev(k["edges"])
    out, attr = filter_adj(e, dev(k["perm"]), edge_attr=torch.arange(len(k["edges"]), device="cuda"))
    assert out.tolist() == k["out"] and attr.tolist() == [0, 1, 3, 4, 12]
    out, _ = filter_adj(e, dev(k["perm"]), num_nodes=50)
    assert out.tolist() == k["out"]
    rng = np.random.default_rng(2)
    e2 = rng.integers(0, 1000, (5000, 2))
    perm = rng.choice(1000, 300, replace=False)
    out, _ = filter_adj(dev(e2), dev(perm))
    assert out.cpu().numpy().tolist() == P.filter_adj(e2, perm).tolist()
    k = kat["graph_norm"]
    g = pgl.Graph.disjoint([pgl.Graph(edges=gg["edges"], num_nodes=gg["num_nodes"]) for gg in k["graphs"]]).tensor()
    f = dev(np.array(k["feature"], np.float32))
    assert pgl.nn.functional.graph_norm(g, f).tolist() == k["out"]
    assert pgl.nn.GraphNorm()(g, f).tolist() == k["out"]


# ---- attention readout --------------------------------------------------------------------------------------------

def readout_bound(x, sizes):
    """fp32 error bound of the readout: every output is a convex combination, accumulated by fma in chunks of at most
    2048 rows and merged over ceil(n / 2048) partials; each term carries an exp rounding (a few ulp) and a product
    rounding, so |out - exact| <= (2048 + chunks + 16) * 2^-24 * max|x| with a factor 4 of headroom for exp."""
    chunks = max(1, int(math.ceil(max(sizes) / 2048)))
    return 4 * (2048 + chunks + 16) * 2.0 ** -24 * float(np.abs(x).max())


@pytest.mark.parametrize("mode", ["gate", "query"])
@pytest.mark.parametrize("D", [3, 300])
def test_attn_readout_vs_oracle(pgl, mode, D):
    rng = np.random.default_rng(D)
    sizes = [0, 1, 2, 7, 2047, 2048, 2049, 5000, 0, 13]
    if D == 3:
        sizes.append(1_000_000)
    n = int(sum(sizes))
    x = rng.standard_normal((n, D)).astype(np.float32)
    ip = indptr_of(sizes)
    if mode == "gate":
        gate = (3 * rng.standard_normal(n)).astype(np.float32)
        out, lse = pgl.ops.attn_readout(dev(x), ip, gate=dev(gate), return_lse=True)
        want, wl = P.attn_readout(x, ip.cpu().numpy(), gate=gate, indptr=True)
    else:
        q = (rng.standard_normal((len(sizes), D)) / math.sqrt(D)).astype(np.float32)
        out, lse = pgl.ops.attn_readout(dev(x), ip, query=dev(q), return_lse=True)
        want, wl = P.attn_readout(x, ip.cpu().numpy(), query=q, indptr=True)
    err = np.abs(out.cpu().numpy() - want).max()
    assert err <= readout_bound(x, sizes), err
    lse = lse.cpu().numpy()
    fin = np.isfinite(wl)
    assert (lse[~fin] == -np.inf).all() and np.abs(lse[fin] - wl[fin]).max() <= 1e-5 * (1 + np.abs(wl[fin]).max())
    assert (out.cpu().numpy()[np.array(sizes) == 0] == 0).all()


def test_attn_readout_overflow_kat(pgl, kat):
    k = kat["segment_softmax_overflow"]
    out = pgl.ops.attn_readout(torch.eye(2, device="cuda"), indptr_of([2]), gate=dev(np.float32(k["scores"])))
    assert out.tolist() == [k["weights"]]


@pytest.mark.parametrize("mode", ["gate", "query"])
def test_attn_readout_deterministic_and_position_free(pgl, mode):
    rng = np.random.default_rng(21)
    D = 64
    g1 = rng.standard_normal((37, D)).astype(np.float32)
    g2 = rng.standard_normal((5000, D)).astype(np.float32)
    big = rng.standard_normal((9000, D)).astype(np.float32)
    s1, s2, sb = (rng.standard_normal(len(a)).astype(np.float32) for a in (g1, g2, big))
    q1, q2, qb = (rng.standard_normal(D).astype(np.float32) / 8 for _ in range(3))

    def run(parts):
        x = np.concatenate([p[0] for p in parts])
        ip = indptr_of([len(p[0]) for p in parts])
        if mode == "gate":
            return pgl.ops.attn_readout(dev(x), ip, gate=dev(np.concatenate([p[1] for p in parts])))
        return pgl.ops.attn_readout(dev(x), ip, query=dev(np.stack([p[2] for p in parts])))

    a = run([(g1, s1, q1), (big, sb, qb), (g2, s2, q2)])
    b = run([(g2, s2, q2), (g1, s1, q1)])
    c = run([(g1, s1, q1)])
    a2 = run([(g1, s1, q1), (big, sb, qb), (g2, s2, q2)])
    assert torch.equal(a, a2)
    assert torch.equal(a[0], b[1]) and torch.equal(a[2], b[0]) and torch.equal(a[0], c[0])


def test_attn_readout_one_launch_below_chunk(pgl):
    rng = np.random.default_rng(3)
    sizes = rng.integers(10, 41, 256)
    x = dev(rng.standard_normal((int(sizes.sum()), 300)).astype(np.float32)).requires_grad_(True)
    gate = dev(rng.standard_normal(int(sizes.sum())).astype(np.float32)).requires_grad_(True)
    ip = indptr_of(sizes)
    pgl.ops.segment_max_len(ip)
    l0 = pgl.ops.launch_count()
    with torch.no_grad():
        pgl.ops.attn_readout(x, ip, gate=gate)
    assert pgl.ops.launch_count() - l0 == 1
    l0 = pgl.ops.launch_count()
    pgl.ops.attn_readout(x, ip, gate=gate).sum().backward()
    assert pgl.ops.launch_count() - l0 == 2


def torch_reference_readout(x, ids, B, gate=None, query=None):
    """The reference composition (pool.py:139-142, 173-178) in torch ops: score, segment softmax, segment sum."""
    if gate is None:
        s = (x * query[ids]).sum(-1)
    else:
        s = gate.reshape(-1)
    m = torch.full((B,), -torch.inf, dtype=x.dtype, device=x.device).scatter_reduce(0, ids, s, "amax")
    e = torch.exp(s - m[ids])
    den = torch.zeros(B, dtype=x.dtype, device=x.device).index_add(0, ids, e)
    a = (e / den[ids]).unsqueeze(1)
    return torch.zeros(B, x.shape[1], dtype=x.dtype, device=x.device).index_add(0, ids, a * x)


@pytest.mark.parametrize("mode", ["gate", "query"])
@pytest.mark.parametrize("sizes", [[1, 0, 5, 30, 2], [3, 4100, 0, 7, 2049]])
def test_attn_readout_backward_vs_float64(pgl, mode, sizes):
    rng = np.random.default_rng(5)
    D = 24
    n, B = int(sum(sizes)), len(sizes)
    x64 = torch.tensor(rng.standard_normal((n, D)), device="cuda")
    s64 = torch.tensor(rng.standard_normal(n), device="cuda")
    q64 = torch.tensor(rng.standard_normal((B, D)) / 4, device="cuda")
    g64 = torch.tensor(rng.standard_normal((B, D)), device="cuda")
    ids = torch.as_tensor(ids_of(sizes)).cuda()
    leaves64 = [x64.clone().requires_grad_(True), (s64 if mode == "gate" else q64).clone().requires_grad_(True)]
    kw = {"gate": leaves64[1]} if mode == "gate" else {"query": leaves64[1]}
    (torch_reference_readout(leaves64[0], ids, B, **kw) * g64).sum().backward()
    leaves = [t.detach().float().requires_grad_(True) for t in leaves64]
    kw = {"gate": leaves[1]} if mode == "gate" else {"query": leaves[1]}
    (pgl.ops.attn_readout(leaves[0], indptr_of(sizes), **kw) * g64.float()).sum().backward()
    for got, want in zip(leaves, leaves64):
        w = want.grad
        err = (got.grad.double() - w).abs().max().item()
        assert err <= 2e-5 * (1 + w.abs().max().item()), err


def test_attn_readout_float64_and_half_dtypes(pgl):
    rng = np.random.default_rng(6)
    sizes = [3, 0, 9]
    x = torch.tensor(rng.standard_normal((12, 8)), device="cuda")
    gate = torch.tensor(rng.standard_normal(12), device="cuda")
    ip = indptr_of(sizes)
    out = pgl.ops.attn_readout(x, ip, gate=gate)
    assert out.dtype == torch.float64
    want, _ = P.attn_readout(x.cpu().numpy(), ip.cpu().numpy(), gate=gate.cpu().numpy(), indptr=True)
    assert np.abs(out.cpu().numpy() - want).max() <= 1e-5
    out16 = pgl.ops.attn_readout(x.to(torch.bfloat16), ip, gate=gate.to(torch.bfloat16))
    assert out16.dtype == torch.bfloat16


# ---- layers -------------------------------------------------------------------------------------------------------

def three_graphs(pgl):
    return pgl.Graph.disjoint([pgl.Graph(num_nodes=i, edges=[(0, 0)]) for i in [3, 2, 1]]).tensor()


DATA = [[1, 2, 3], [3, 2, 1], [4, 5, 6], [1, 2, 3], [3, 2, 1], [1, 2, 3]]
MIXED = [[4, 5, 6], [3, 2, 1], [1, 2, 3], [3, 2, 1], [1, 2, 3], [1, 2, 3]]


def test_reference_pool_permutation_invariance(pgl):
    torch.manual_seed(0)
    g = three_graphs(pgl)
    a, b = dev(np.float32(DATA)), dev(np.float32(MIXED))
    for layer in (pgl.nn.GlobalAttention(pgl.nn.Linear(3, 1)), pgl.nn.Set2Set(3, 2).cuda(),
                  pgl.nn.GraphPool("mean")):
        layer = layer.cuda()
        np.testing.assert_almost_equal(layer(g, a).detach().cpu().numpy(), layer(g, b).detach().cpu().numpy(), 5)
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        pgl.nn.GraphPool("sum")(g, a, pool_type="mean")
    assert any("discarded" in str(x.message) for x in w)


def test_reference_gmt_and_sag_pool(pgl):
    torch.manual_seed(1)
    rng = np.random.default_rng(1)
    g1 = pgl.Graph(edges=[(0, 1), (1, 2), (3, 4)], num_nodes=5,
                   node_feat={"nfeat": rng.standard_normal((5, 12)).astype(np.float32)})
    g2 = pgl.Graph(edges=[(0, 1), (1, 2), (3, 4), (5, 2), (0, 5)], num_nodes=6,
                   node_feat={"nfeat": rng.standard_normal((6, 12)).astype(np.float32)})
    g = pgl.Graph.disjoint([g1, g2]).tensor()
    gmt = pgl.nn.GraphMultisetTransformer(12, 12, 12, num_nodes=5).cuda()
    out = gmt(g, g.node_feat["nfeat"])
    assert out.shape == (2, 12)
    gmt_ln = pgl.nn.GraphMultisetTransformer(12, 12, 12, num_nodes=5, layer_norm=True).cuda()
    assert gmt_ln(g, g.node_feat["nfeat"]).shape == (2, 12)
    # SAGPool, tests/test_pool.py:119-146
    x = torch.randn(8, 4, device="cuda")
    e = torch.tensor([[0, 1, 2, 3, 4, 5, 5, 6, 6, 7], [1, 0, 3, 4, 2, 6, 7, 7, 5, 6]], device="cuda").t()
    gs = pgl.Graph(num_nodes=8, edges=e, node_feat={"attr": x},
                   _graph_node_index=torch.tensor([0, 2, 5, 8], device="cuda"), _num_graph=3).tensor()
    out, batch, pooled = pgl.nn.SAGPool(4, 0.5, pgl.nn.GCNConv).cuda()(gs, x)
    assert out.shape[0] == math.ceil(0.5 * 2) + math.ceil(0.5 * 3) + math.ceil(0.5 * 3)
    assert pooled.num_graph == 3 and pooled.edges.shape[1] == 2
    assert pooled.graph_node_id.tolist() == batch.tolist()
    out2, _, _ = pgl.nn.SAGPool(4, 0.5).cuda()(gs, x)     # gnn=None: GCNConv
    assert out2.shape == out.shape


def test_global_attention_and_set2set_vs_torch_restatement(pgl):
    torch.manual_seed(2)
    sizes = [5, 1, 17, 3]
    g = batch_graph(pgl, sizes)
    x = torch.randn(sum(sizes), 16, device="cuda")
    ids = g.graph_node_id.long()
    gate_nn, feat_nn = pgl.nn.Linear(16, 1).cuda(), pgl.nn.Linear(16, 8).cuda()
    ga = pgl.nn.GlobalAttention(gate_nn, feat_nn)
    want = torch_reference_readout(feat_nn(x), ids, 4, gate=gate_nn(x))
    assert (ga(g, x) - want).abs().max().item() <= 1e-5
    s2s = pgl.nn.Set2Set(16, 3).cuda()
    seen = []
    s2s.lstm.register_forward_hook(lambda m, inp, out: seen.append(inp[0].detach().clone()))
    got = s2s(g, x)
    # the reference's q_star is never updated: every LSTM input is zeros
    assert len(seen) == 3 and all(bool((t == 0).all()) for t in seen)
    h = (torch.zeros(1, 4, 16, device="cuda"), torch.zeros(1, 4, 16, device="cuda"))
    for _ in range(3):
        q, h = s2s.lstm(torch.zeros(1, 4, 32, device="cuda"), h)
        q = q.reshape(4, 16)
        want = torch.cat([q, torch_reference_readout(x, ids, 4, query=q)], -1)
    assert got.shape == (4, 32) and (got - want).abs().max().item() <= 1e-5


def test_sag_pool_vs_torch_restatement(pgl):
    torch.manual_seed(3)
    sizes = [6, 9, 4, 11]
    g = batch_graph(pgl, sizes, seed=3)
    x = torch.randn(sum(sizes), 8, device="cuda")
    sag = pgl.nn.SAGPool(8, ratio=0.5).cuda()
    out, batch, pooled = sag(g, x)
    score = torch.tanh(sag.gnn(g, x).reshape(-1))
    ids = g.graph_node_id.long().cpu().numpy()
    perm = P.segment_topk_perm(score.detach().cpu().numpy(), ids, 0.5)
    want = x[torch.as_tensor(perm).cuda()] * score[torch.as_tensor(perm).cuda()].reshape(-1, 1)
    assert torch.allclose(out, want, atol=1e-6)
    assert batch.tolist() == ids[perm].tolist()
    want_edges = P.filter_adj(g.edges.cpu().numpy(), perm, num_nodes=sum(sizes))
    assert pooled.edges.cpu().numpy().tolist() == want_edges.tolist()
    assert pooled.num_nodes.item() == len(perm)


def test_gmt_mask_quirk(pgl):
    """A real node whose features sum to 0 is masked like padding (gmt_pool.py:285)."""
    torch.manual_seed(4)
    g = batch_graph(pgl, [3, 2], seed=4)
    gmt = pgl.nn.GraphMultisetTransformer(4, 8, 8, num_nodes=3).cuda()
    x = torch.randn(5, 4, device="cuda")
    from pgl_b200.utils.transform import to_dense_batch
    h = gmt.lin1(x)
    batch_x, pad = to_dense_batch(h, g)
    mask = (batch_x.sum(-1) == 0)
    assert mask.tolist() == pad.tolist()
    with torch.no_grad():
        gmt.lin1.weight.zero_()
        gmt.lin1.bias.zero_()
    bx, pad = to_dense_batch(gmt.lin1(x), g)
    assert bool((bx.sum(-1) == 0).all()) and not bool(pad.all())


def test_graph_classification_training(pgl):
    """GINConv + SAGPool + GlobalAttention (and Set2Set) readout on seeded synthetic graphs: two classes that differ
    in structure (rings vs stars) and node-feature mean; the loss falls and training accuracy exceeds 0.9."""
    rng = np.random.default_rng(0)
    torch.manual_seed(0)

    def make(label, n):
        if label == 0:
            e = [(i, (i + 1) % n) for i in range(n)]
        else:
            e = [(0, i) for i in range(1, n)]
        e = e + [(b, a) for a, b in e]
        feat = (rng.standard_normal((n, 8)) + (0.5 if label else -0.5)).astype(np.float32)
        return pgl.Graph(edges=e, num_nodes=n, node_feat={"h": feat})

    labels = rng.integers(0, 2, 128)
    graphs = [make(int(y), int(rng.integers(6, 20))) for y in labels]
    g = pgl.Graph.disjoint(graphs).tensor()
    y = torch.as_tensor(labels).cuda()

    for readout in ("attention", "set2set"):
        class Net(torch.nn.Module):
            def __init__(self):
                super().__init__()
                self.gin = pgl.nn.GINConv(8, 32, activation="relu")
                self.pool = pgl.nn.SAGPool(32, ratio=0.5)
                if readout == "attention":
                    self.read = pgl.nn.GlobalAttention(pgl.nn.Linear(32, 1))
                    self.head = pgl.nn.Linear(32, 2)
                else:
                    self.read = pgl.nn.Set2Set(32, 2)
                    self.head = pgl.nn.Linear(64, 2)

            def forward(self, g, x):
                h = torch.relu(self.gin(g, x))
                h, _, pg = self.pool(g, h)
                return self.head(self.read(pg, h))

        net = Net().cuda()
        opt = torch.optim.Adam(net.parameters(), lr=0.01)
        losses = []
        for _ in range(60):
            opt.zero_grad()
            loss = torch.nn.functional.cross_entropy(net(g, g.node_feat["h"]), y)
            loss.backward()
            opt.step()
            losses.append(loss.item())
        acc = (net(g, g.node_feat["h"]).argmax(1) == y).float().mean().item()
        assert losses[-1] < 0.5 * losses[0], (readout, losses[0], losses[-1])
        assert acc > 0.9, (readout, acc)
