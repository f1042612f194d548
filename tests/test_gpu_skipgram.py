"""Skip-gram pairs and alias sampling on the device (csrc/skipgram.cu through pgl_b200.sampling): bit for bit against
the host entry pglb_skipgram_host on walks from random_walk, node2vec_walk and metapath_randomwalk over RMAT 2^16 graphs
with sinks, at batch sizes where the multi-block scan engages; list and tensor input; seeds; the int64 pair offsets
past 2^32; alias draws against the numpy replay and a chi-square test against outdegree^0.75; the launch count; and
an end-to-end DeepWalk on Cora whose probe accuracy matches the numpy reference pipeline's."""
import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

from oracle import oracle_skipgram as S

pytestmark = pytest.mark.gpu

N16 = 1 << 16


@pytest.fixture(scope="module")
def pgl():
    import pgl_b200
    torch.cuda.set_device(0)
    return pgl_b200


def ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def rmat_edges(scale, e, seed):
    """RMAT (0.57, 0.19, 0.19, 0.05), duplicates and self-loops kept; many nodes have no out-edge."""
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    src = torch.zeros(e, dtype=torch.int64, device="cuda")
    dst = torch.zeros(e, dtype=torch.int64, device="cuda")
    for _ in range(scale):
        r = torch.rand(e, generator=gen, device="cuda")
        src = src * 2 + (r >= 0.76).to(torch.int64)
        dst = dst * 2 + (((r >= 0.57) & (r < 0.76)) | (r >= 0.95)).to(torch.int64)
    return torch.stack([src, dst], 1).contiguous()


@pytest.fixture(scope="module")
def graphs(pgl):
    edges = rmat_edges(16, 8 * N16, 5)
    g = pgl.Graph(edges=edges, num_nodes=N16)
    half = edges.shape[0] // 2
    hg = pgl.HeterGraph(edges={"r0": edges[:half].cpu().numpy(), "r1": edges[half:].cpu().numpy()}, num_nodes=N16,
                        node_types=np.zeros(N16, np.int64)).tensor()
    return g, hg, edges


def host_pairs(lib, walks, win_size, seed):
    walks = np.ascontiguousarray(walks, np.int64)
    B, L = walks.shape
    offsets = np.empty(B + 1, np.int64)
    assert lib.pglb_skipgram_host(ptr(walks), B, L, win_size, seed, ptr(offsets), None, None) == 0
    src = np.empty(offsets[B], np.int64)
    pos = np.empty(offsets[B], np.int64)
    assert lib.pglb_skipgram_host(ptr(walks), B, L, win_size, seed, ptr(offsets), ptr(src), ptr(pos)) == 0
    return src, pos


def make_walks(pgl, graphs, kind, B, L, seed):
    g, hg, _ = graphs
    gen = torch.Generator(device="cuda")
    gen.manual_seed(B * 7 + L)
    nodes = torch.randint(0, N16, (B,), generator=gen, device="cuda")
    if kind == "random":
        return pgl.sampling.random_walk(g, nodes, L, seed=seed)
    if kind == "node2vec":
        return pgl.sampling.node2vec_walk(g, nodes, L - 1, p=0.5, q=2.0, seed=seed)
    return pgl.sampling.metapath_randomwalk(hg, nodes, "r0-r1", L, seed=seed)


# (walk kind, B, L, win_size): the large batches with short walks and small windows
CASES = [("random", 1, 40, 10), ("random", 512, 40, 10), ("node2vec", 512, 130, 64), ("metapath", 512, 40, 3),
         ("random", 512, 1, 3), ("node2vec", 512, 2, 1), ("metapath", 100_000, 40, 10), ("random", 100_000, 130, 3),
         ("node2vec", 100_000, 2, 64), ("random", 1_000_000, 10, 3), ("metapath", 1_000_000, 2, 1),
         ("random", 1_000_000, 40, 1)]


@pytest.mark.parametrize("kind,B,L,win_size", CASES)
def test_device_pairs_are_the_host_entry(pgl, graphs, kind, B, L, win_size):
    from pgl_b200 import _lib
    walks = make_walks(pgl, graphs, kind, B, L, seed=B + L)
    assert walks.shape == (B, L)
    if L > 1 and B >= 512:
        assert (walks[:, -1] < 0).any()   # sinks: padded rows
    for seed in (0, 2 ** 64 - 1):
        src, pos = pgl.sampling.skip_gram_pairs(walks, win_size, seed=seed)
        assert src.is_cuda and src.dtype == torch.int64 and pos.dtype == torch.int64
        hs, hp = host_pairs(_lib.lib, walks.cpu().numpy(), win_size, seed)
        assert np.array_equal(src.cpu().numpy(), hs) and np.array_equal(pos.cpu().numpy(), hp), (kind, B, L, seed)
        if B == 1:
            rs, rp = S.replay_skipgram(walks.cpu().numpy(), S.skipgram_windows(B, L, win_size, seed))
            assert np.array_equal(hs, rs) and np.array_equal(hp, rp)
        del src, pos
    torch.cuda.empty_cache()


def test_list_input_is_tensor_input(pgl, graphs):
    g, _, e = graphs
    gn = pgl.Graph(edges=e.cpu().numpy(), num_nodes=N16)
    nodes = np.random.default_rng(1).integers(0, N16, 700)
    lists = pgl.sampling.random_walk(gn, nodes, 30, seed=9)
    tens = pgl.sampling.random_walk(g, torch.as_tensor(nodes).cuda(), 30, seed=9)
    s, p = pgl.sampling.skip_gram_pairs(lists, 5, seed=3)
    assert isinstance(s, np.ndarray) and s.dtype == np.int64
    ts, tp = pgl.sampling.skip_gram_pairs(tens, 5, seed=3)
    assert np.array_equal(s, ts.cpu().numpy()) and np.array_equal(p, tp.cpu().numpy())


def test_seeds(pgl, graphs):
    walks = make_walks(pgl, graphs, "random", 4096, 40, seed=1)
    a = pgl.sampling.skip_gram_pairs(walks, 10, seed=123)
    b = pgl.sampling.skip_gram_pairs(walks, 10, seed=123)
    c = pgl.sampling.skip_gram_pairs(walks, 10, seed=124)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert a[0].numel() != c[0].numel() or not torch.equal(a[1], c[1])
    np.random.seed(5)
    d = pgl.sampling.skip_gram_pairs(walks, 10)
    np.random.seed(5)
    e = pgl.sampling.skip_gram_pairs(walks, 10)
    assert torch.equal(d[1], e[1])


def test_count_offsets_past_2_32(pgl):
    """2^13 walks of 1 024 distinct nodes with win_size = 2^20: nearly every window spans the walk, so the total is
    close to B L (L - 1) = 8.6e9, past 2^32.  Only the count runs; each walk's count is the sum over its centres of
    min(L - 1, i + w) - max(0, i - w) with the replayed windows (distinct nodes: every other position pairs)."""
    from pgl_b200 import _lib, ops
    B, L, win, seed = 1 << 13, 1024, 1 << 20, 77
    walks = torch.arange(B * L, dtype=torch.int64, device="cuda").reshape(B, L)
    offsets = torch.empty(B + 1, dtype=torch.int64, device="cuda")
    need = ctypes.c_size_t(0)
    assert _lib.lib.pglb_skipgram_count_ws(B, ctypes.byref(need)) == 0
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    _lib.check(_lib.lib.pglb_skipgram_count(ops._ptr(walks), B, L, win, seed, ops._ptr(offsets), ops._ptr(ws),
                                            ws.numel(), ops._stream()))
    w = S.skipgram_windows(B, L, win, seed)
    i = np.arange(L)[None, :]
    per_walk = (np.minimum(L - 1, i + w) - np.maximum(0, i - w)).sum(1)
    want = np.concatenate([[0], np.cumsum(per_walk)])
    assert np.array_equal(offsets.cpu().numpy(), want)
    assert want[-1] > 2 ** 32 and want[-1] > 0.99 * B * L * (L - 1)


@pytest.mark.parametrize("n", [1, 2, 7, 1000, 10 ** 6])
def test_alias_sample_is_the_replay(pgl, n):
    rng = np.random.default_rng(n)
    w = rng.pareto(1.0, n) * (rng.random(n) < 0.9)
    w[0] += 1.0
    alias, events = pgl.sampling.alias_table(w)
    for seed in (0, 2 ** 64 - 1):
        got = pgl.sampling.alias_sample(torch.from_numpy(alias).cuda(), torch.from_numpy(events).cuda(), (1000, 300),
                                        seed=seed)
        assert got.shape == (1000, 300) and got.is_cuda and got.dtype == torch.int64
        want = S.alias_draws(alias, events, 300_000, seed).reshape(1000, 300)
        assert np.array_equal(got.cpu().numpy(), want)
        got_np = pgl.sampling.alias_sample(alias, events, 300_000, seed=seed)
        assert isinstance(got_np, np.ndarray) and np.array_equal(got_np, want.reshape(-1))


def test_alias_sample_distribution(pgl, graphs):
    """10^7 draws against outdegree^0.75 of the RMAT graph: zero-weight nodes never drawn, chi-square on the rest
    (bins with an expected count below 5 pooled)."""
    g, _, _ = graphs
    w = g.outdegree().double() ** 0.75
    alias, events = pgl.sampling.alias_table(w)
    assert alias.is_cuda and events.is_cuda
    count = 10 ** 7
    draws = pgl.sampling.alias_sample(alias, events, count, seed=31)
    obs = torch.bincount(draws, minlength=N16).cpu().numpy()
    p = (w / w.sum()).cpu().numpy()
    assert obs.sum() == count and obs[p == 0].sum() == 0
    exp = p * count
    big = exp >= 5
    small = ~big & (p > 0)
    o, ex = obs[big], exp[big]
    if small.any():
        o, ex = np.r_[o, obs[small].sum()], np.r_[ex, exp[small].sum()]
    assert stats.chisquare(o, ex).pvalue > 1e-4


def test_launch_count(pgl, graphs):
    walks = make_walks(pgl, graphs, "random", 512, 40, seed=2)
    alias, events = pgl.sampling.alias_table(torch.ones(100, device="cuda"))
    torch.cuda.synchronize()
    before = pgl.ops.launch_count()
    src, _ = pgl.sampling.skip_gram_pairs(walks, 10, seed=1)
    assert pgl.ops.launch_count() - before == 5   # count, the three scan launches, fill
    before = pgl.ops.launch_count()
    pgl.sampling.alias_sample(alias, events, (src.numel(), 20), seed=1)
    assert pgl.ops.launch_count() - before == 1


# ---- end-to-end DeepWalk on Cora -------------------------------------------------------------------------------

DW_STEPS, DW_BATCH, DW_WALK, DW_WIN, DW_NEG, DW_DIM = 200, 512, 40, 5, 5, 64
# Probe-accuracy floor.  Measured on an H100 80GB HBM3 (700 W): device pipeline 0.796, numpy reference pipeline 0.783
# (DESIGN.md section 4.17); set below both so it catches a broken pipeline, not the run-to-run spread of the
# embeddings' atomic gradient sums.
DW_FLOOR = 0.75


def _train(pairs_of_batch, num_nodes, seed):
    """skip-gram with negative sampling: torch Embeddings, Adam, a fixed number of steps"""
    torch.manual_seed(seed)
    emb = torch.nn.Embedding(num_nodes, DW_DIM).cuda()
    ctx = torch.nn.Embedding(num_nodes, DW_DIM).cuda()
    torch.nn.init.uniform_(emb.weight, -0.5 / DW_DIM, 0.5 / DW_DIM)
    torch.nn.init.zeros_(ctx.weight)
    opt = torch.optim.Adam(list(emb.parameters()) + list(ctx.parameters()), lr=0.01)
    for step in range(DW_STEPS):
        src, pos, neg = pairs_of_batch(step)
        u = emb(src)
        lp = torch.nn.functional.logsigmoid((u * ctx(pos)).sum(-1))
        ln = torch.nn.functional.logsigmoid(-(u[:, None, :] * ctx(neg)).sum(-1)).sum(-1)
        loss = -(lp + ln).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
    return emb.weight.detach()


def _probe(x, y, seed):
    """logistic regression on the normalised embeddings: a seeded 50 / 50 split, full-batch Adam"""
    x = torch.nn.functional.normalize(x, dim=1)
    n = x.shape[0]
    perm = torch.from_numpy(np.random.default_rng(seed).permutation(n)).cuda()
    tr, te = perm[:n // 2], perm[n // 2:]
    torch.manual_seed(seed)
    lin = torch.nn.Linear(x.shape[1], int(y.max()) + 1).cuda()
    opt = torch.optim.Adam(lin.parameters(), lr=0.05)
    for _ in range(300):
        loss = torch.nn.functional.cross_entropy(lin(x[tr]), y[tr])
        opt.zero_grad()
        loss.backward()
        opt.step()
    return float((lin(x[te]).argmax(1) == y[te]).float().mean())


def test_deepwalk_on_cora(pgl):
    import os

    from oracle import oracle as O
    import pgl.graph_kernel as gk
    cora = O.load_cora(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "cora.npz"))
    n, edges = cora["num_nodes"], cora["edges"]
    edges = np.concatenate([edges, edges[:, ::-1]])   # undirected, as the reference's deepwalk example builds it
    g = pgl.Graph(edges=edges, num_nodes=n).tensor()
    y = torch.from_numpy(cora["y"]).cuda()
    deg = np.bincount(edges[:, 0], minlength=n).astype(np.float64)
    alias, events = pgl.sampling.alias_table(torch.from_numpy(deg ** 0.75).cuda())
    rng = np.random.default_rng(0)
    batches = [rng.integers(0, n, DW_BATCH) for _ in range(DW_STEPS)]

    def walks_of(step):
        return pgl.sampling.random_walk(g, torch.from_numpy(batches[step]).cuda(), DW_WALK, seed=1000 + step)

    def device_batch(step):
        src, pos = pgl.sampling.skip_gram_pairs(walks_of(step), DW_WIN, seed=2000 + step)
        neg = pgl.sampling.alias_sample(alias, events, (src.numel(), DW_NEG), seed=3000 + step)
        return src, pos, neg

    np.random.seed(0)

    def numpy_batch(step):
        rows = walks_of(step).cpu().numpy()
        s, p = [], []
        for row in rows:
            a, b = gk.skip_gram_gen_pair(row[row >= 0], DW_WIN)
            s += a
            p += b
        neg = np.random.randint(0, n, (len(s), DW_NEG))
        return (torch.tensor(s, device="cuda"), torch.tensor(p, device="cuda"), torch.from_numpy(neg).cuda())

    acc_dev = _probe(_train(device_batch, n, 0), y, 0)
    acc_ref = _probe(_train(numpy_batch, n, 0), y, 0)
    print("deepwalk cora probe accuracy: device %.4f numpy reference %.4f" % (acc_dev, acc_ref))
    assert acc_dev >= acc_ref - 0.02
    assert acc_dev >= DW_FLOOR
