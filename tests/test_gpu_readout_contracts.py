"""Contracts of the graph-level readouts that need the device: a max_len below the longest segment (attention readout
and top-k) still gives correct results; the chunk split and merge of the readout are exact on integer data; the
pooling layers read the batch's segment CSR once per graph; GraphMultisetTransformer against a torch restatement of
the reference's op order with its quirks (sum-zero mask, softmax over axis 1, ln0 twice), each shown to change the
output; SAGPool's min_score path; graph_norm in 16-bit; filter_adj's id checks."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import oracle_pool as P

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    torch.cuda.set_device(0)
    return pgl_b200


def dev(a, dtype=None):
    return torch.as_tensor(np.asarray(a), dtype=dtype).cuda()


def ids_of(sizes):
    return np.repeat(np.arange(len(sizes)), sizes).astype(np.int64)


def indptr_of(sizes):
    return dev(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64))


def ring_batch(pgl, sizes):
    gs = []
    for n in sizes:
        e = [(j, (j + 1) % n) for j in range(n)] + [((j + 1) % n, j) for j in range(n)] if n > 1 else [(0, 0)]
        gs.append(pgl.Graph(edges=e, num_nodes=n))
    return pgl.Graph.disjoint(gs).tensor()


def torch_reference_readout(x, ids, B, gate=None, query=None):
    s = (x * query[ids]).sum(-1) if gate is None else gate.reshape(-1)
    m = torch.full((B,), -torch.inf, dtype=x.dtype, device=x.device).scatter_reduce(0, ids, s, "amax")
    e = torch.exp(s - m[ids])
    den = torch.zeros(B, dtype=x.dtype, device=x.device).index_add(0, ids, e)
    return torch.zeros(B, x.shape[1], dtype=x.dtype, device=x.device).index_add(0, ids, (e / den[ids]).unsqueeze(1) * x)


# ---- attention readout: understated max_len, exact chunk merge ------------------------------------------------------

@pytest.mark.parametrize("mode", ["gate", "query"])
def test_attn_readout_understated_max_len(pgl, mode):
    """A stale max_len (here 10, for segments of up to 3000 rows) reads every long segment as one chunk: forward and
    every gradient stay correct, in one launch each."""
    rng = np.random.default_rng(1)
    sizes = [3000, 5, 0, 2100, 1]
    n, B, D = sum(sizes), len(sizes), 16
    x64 = torch.tensor(rng.standard_normal((n, D)), device="cuda")
    s64 = torch.tensor(rng.standard_normal(n), device="cuda")
    q64 = torch.tensor(rng.standard_normal((B, D)) / 4, device="cuda")
    g64 = torch.tensor(rng.standard_normal((B, D)), device="cuda")
    ids = torch.as_tensor(ids_of(sizes)).cuda()
    leaves64 = [x64.clone().requires_grad_(True), (s64 if mode == "gate" else q64).clone().requires_grad_(True)]
    kw = {"gate": leaves64[1]} if mode == "gate" else {"query": leaves64[1]}
    want = torch_reference_readout(leaves64[0], ids, B, **kw)
    (want * g64).sum().backward()
    ip = indptr_of(sizes)
    ip._pglb_max_len = 10                       # stale: the longest segment has 3000 rows
    leaves = [t.detach().float().requires_grad_(True) for t in leaves64]
    kw = {"gate": leaves[1]} if mode == "gate" else {"query": leaves[1]}
    l0 = pgl.ops.launch_count()
    out = pgl.ops.attn_readout(leaves[0], ip, **kw)
    (out * g64.float()).sum().backward()
    assert pgl.ops.launch_count() - l0 == 2
    assert (out.double() - want).abs().max().item() <= 1e-5
    for got, w in zip(leaves, leaves64):
        assert torch.isfinite(got.grad).all()
        err = (got.grad.double() - w.grad).abs().max().item()
        assert err <= 2e-5 * (1 + w.grad.abs().max().item()), err


@pytest.mark.parametrize("mode", ["gate", "query"])
def test_attn_readout_chunk_merge_exact(pgl, mode):
    """Scores of 0 and small-integer features make every step exact in fp32 (weights 1, sums below 2^24), so each
    output must equal fl32(sum / n) bit for bit: dropping or double-counting one row anywhere in the chunk split or the
    merge would show."""
    rng = np.random.default_rng(2)
    sizes = [1_000_000, 2048, 2049, 4096, 0, 6001, 1, 37]
    n, B, D = sum(sizes), len(sizes), 4
    x = rng.integers(-1, 3, (n, D)).astype(np.float32)
    ip = indptr_of(sizes)
    kw = {"gate": torch.zeros(n, device="cuda")} if mode == "gate" else {"query": torch.zeros(B, D, device="cuda")}
    out, lse = pgl.ops.attn_readout(dev(x), ip, return_lse=True, **kw)
    ipn = ip.cpu().numpy()
    want = np.zeros((B, D), np.float32)
    for g in range(B):
        if sizes[g]:
            want[g] = (x[ipn[g]:ipn[g + 1]].astype(np.float64).sum(0) / sizes[g]).astype(np.float32)
    assert np.array_equal(out.cpu().numpy(), want)
    lse = lse.cpu().numpy()
    for g in range(B):
        if sizes[g] == 0:
            assert lse[g] == -np.inf
        else:
            assert abs(lse[g] - np.log(sizes[g])) <= 2 * np.spacing(np.float32(np.log(sizes[g]))) + 1e-7


def test_topk_understated_max_len(pgl):
    """The fill entry with a max_len below a segment longer than the shared array ranks that segment from global
    memory: the same perm as the oracle."""
    from pgl_b200 import _lib
    rng = np.random.default_rng(3)
    sizes = np.array([3000, 40, 0, 2500, 7])
    ids = ids_of(sizes)
    s_np = rng.integers(-3, 4, ids.size).astype(np.float32)
    s = dev(s_np)
    ip = indptr_of(sizes)
    B, N = len(sizes), int(ids.size)
    offsets = torch.empty(B + 1, dtype=torch.int64, device="cuda")
    info = torch.empty(2, dtype=torch.int64, device="cuda")
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    vp = lambda t: ctypes.c_void_p(t.data_ptr())  # noqa: E731
    _lib.check(_lib.lib.pglb_segment_topk_count(vp(ip), B, 0.4, 0, vp(offsets), vp(info), st))
    got = torch.empty(int(info[0].item()), dtype=torch.int64, device="cuda")
    _lib.check(_lib.lib.pglb_segment_topk_fill(vp(s), N, vp(ip), B, vp(offsets), 50, vp(got), None, 0, st))
    assert got.cpu().numpy().tolist() == P.segment_topk_perm(s_np, ids, 0.4).tolist()


# ---- layers -------------------------------------------------------------------------------------------------------

def test_layers_read_the_batch_csr_once(pgl):
    torch.manual_seed(0)
    g = ring_batch(pgl, [5, 1, 17, 3])
    x = torch.randn(26, 16, device="cuda")
    ga = pgl.nn.GlobalAttention(pgl.nn.Linear(16, 1)).cuda()
    s2s = pgl.nn.Set2Set(16, 3).cuda()
    with torch.no_grad():
        first = ga(g, x)
        l0 = pgl.ops.launch_count()
        again = ga(g, x)
        assert pgl.ops.launch_count() - l0 == 1          # the readout alone: no ids, no indptr, no read back
        l0 = pgl.ops.launch_count()
        s2s(g, x)
        assert pgl.ops.launch_count() - l0 == 3          # one readout per iteration
    assert torch.equal(first, again)
    # trailing empty graphs get no output row, as with the reference's last id + 1 segments
    ge = pgl.Graph(num_nodes=4, edges=torch.zeros((0, 2), dtype=torch.int64, device="cuda"),
                   _graph_node_index=torch.tensor([0, 0, 3, 4, 4], device="cuda"), _num_graph=4).tensor()
    assert ga(ge, torch.randn(4, 16, device="cuda")).shape == (3, 16)


def dense(x, graph):
    ids = graph.graph_node_id.long()
    B = int(ids.max()) + 1
    counts = torch.bincount(ids, minlength=B)
    pos = torch.arange(ids.numel(), device=ids.device) - (torch.cumsum(counts, 0) - counts)[ids]
    out = torch.zeros(B, int(counts.max()), x.shape[1], dtype=x.dtype, device=x.device)
    out[ids, pos] = x
    return out, pos, counts


def lin(layer, x):
    return x @ layer.weight + layer.bias


def mab_ref(mab, Q, K, graph, mask, axis, use_ln1):
    """reference gmt_pool.py:77-109 in torch ops with the module's weights."""
    Q = lin(mab.proj_q, Q)
    if graph is not None:
        g, x = graph
        K, V = dense(mab.layer_k(g, x), g)[0], dense(mab.layer_v(g, x), g)[0]
    else:
        K, V = lin(mab.layer_k, K), lin(mab.layer_v, K)
    hd = mab.dim_V // mab.num_heads
    Q_, K_, V_ = (torch.cat(t.split(hd, 2), 0) for t in (Q, K, V))
    score = Q_.bmm(K_.transpose(1, 2)) / math.sqrt(mab.dim_V)
    if mask is not None:
        score = torch.cat([mask] * mab.num_heads, 0).reshape(K_.shape[0], K_.shape[1]).unsqueeze(1) + score
    out = torch.cat((Q_ + torch.softmax(score, axis).bmm(V_)).split(Q.shape[0], 0), 2)
    if mab.layer_norm:
        out = mab.ln0(out)
    out = out + torch.relu(lin(mab.proj_o, out))
    if mab.layer_norm:
        out = (mab.ln1 if use_ln1 else mab.ln0)(out)
    return out


def gmt_ref(gmt, graph, x, mask_mode="sum_zero", axis=1, use_ln1=False):
    """reference gmt_pool.py:283-291 in torch ops with the module's weights."""
    from pgl_b200.nn.gmt_pool import PMA
    x = lin(gmt.lin1, x)
    bx, pos, counts = dense(x, graph)
    if mask_mode == "sum_zero":
        m = bx.sum(-1) == 0
    else:   # padding only
        m = torch.arange(bx.shape[1], device=x.device).unsqueeze(0) >= counts.unsqueeze(1)
    mask = m.to(bx.dtype).unsqueeze(0) * -1e9
    for name, pool in zip(gmt.pool_sequences, gmt.pools):
        g = (graph, x) if name == "GMPool_G" else None
        Q = pool.Q_S.expand(bx.shape[0], pool.num_seeds, pool.dim) if isinstance(pool, PMA) else bx
        bx = mab_ref(pool.mab, Q, bx, g, mask, axis, use_ln1)
        mask = None
    return lin(gmt.lin2, bx.squeeze(1))


@pytest.mark.parametrize("layer_norm", [False, True])
def test_gmt_vs_torch_restatement(pgl, layer_norm):
    torch.manual_seed(5)
    g = ring_batch(pgl, [5, 6, 4])
    x = torch.randn(15, 12, device="cuda")
    x[2] = 0.0                                           # a real node whose lin1 output is all zeros
    gmt = pgl.nn.GraphMultisetTransformer(12, 12, 12, num_nodes=5, layer_norm=layer_norm).cuda()
    with torch.no_grad():
        gmt.lin1.bias.zero_()
        if layer_norm:
            for pool in gmt.pools:
                pool.mab.ln1.weight.fill_(2.0)
                pool.mab.ln1.bias.fill_(0.5)
        out = gmt(g, x)
        want = gmt_ref(gmt, g, x)
        assert out.shape == (3, 12)
        assert (out - want).abs().max().item() <= 1e-4
        # each kept quirk decides outputs: the padding-only mask, softmax over the keys, or ln1 would change them
        assert (out - gmt_ref(gmt, g, x, mask_mode="padding")).abs().max().item() > 1e-3
        assert (out - gmt_ref(gmt, g, x, axis=2)).abs().max().item() > 1e-3
        if layer_norm:
            assert (out - gmt_ref(gmt, g, x, use_ln1=True)).abs().max().item() > 1e-3


def test_sag_pool_min_score(pgl):
    torch.manual_seed(6)
    sizes = [6, 9, 4, 11]
    g = ring_batch(pgl, sizes)
    x = torch.randn(sum(sizes), 8, device="cuda")
    ids = g.graph_node_id.long()
    sag = pgl.nn.SAGPool(8, ratio=0.5, min_score=0.15).cuda()
    out, batch, pooled = sag(g, x)
    raw = sag.gnn(g, x).reshape(-1)
    score = pgl.math.segment_softmax(raw, g.graph_node_id)
    per = [torch.softmax(raw[ids == k], 0) for k in range(len(sizes))]
    assert (score - torch.cat(per)).abs().max().item() <= 1e-6
    _, perm = P.segment_topk(x.cpu().numpy(), score.detach().cpu().numpy(), ids.cpu().numpy(), 0.5, min_score=0.15)
    pt = torch.as_tensor(perm).cuda()
    assert torch.allclose(out, x[pt] * score[pt].reshape(-1, 1), atol=1e-6)
    assert batch.tolist() == ids[pt].tolist() and pooled.num_graph == int(ids[pt].max()) + 1


def test_graph_norm_keeps_16bit_dtype(pgl):
    g = ring_batch(pgl, [3, 4])
    f = torch.randn(7, 5, device="cuda")
    norm = torch.sqrt(torch.tensor([3.0] * 3 + [4.0] * 4, device="cuda")).reshape(-1, 1)
    assert torch.equal(pgl.nn.functional.graph_norm(g, f), f / norm)
    for dt in (torch.bfloat16, torch.float16):
        got = pgl.nn.functional.graph_norm(g, f.to(dt))
        assert got.dtype == dt
        assert torch.equal(got, (f.to(dt).float() / norm).to(dt))


def test_filter_adj_ids(pgl):
    from pgl_b200.utils.transform import filter_adj
    e = dev([[0, 1], [1, 2], [2, 9], [9, 0]])
    out, _ = filter_adj(e, dev([0, 9, 12, 1]))        # 12: a kept isolated node above every edge id
    assert out.tolist() == P.filter_adj([[0, 1], [1, 2], [2, 9], [9, 0]], [0, 9, 12, 1], num_nodes=13).tolist()
    with pytest.raises(ValueError):
        filter_adj(e, dev([0, 12]), num_nodes=10)
    with pytest.raises(ValueError):
        filter_adj(e, dev([-1, 2]))
